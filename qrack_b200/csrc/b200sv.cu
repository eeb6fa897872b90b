// b200sv.cu — C ABI + non-fused kernels of the state-vector core (H100, sm_90a).
//
// What this file replaces in the reference (unitaryfoundation/qrack): the QEngineCUDA host driver
// (src/qengine/cuda.cu) and the non-ALU kernels of src/common/qengine.cu.  Semantics follow QEngineCPU
// (src/qengine/state.cpp), which is the parity oracle; each ABI function cites the lines it mirrors in
// include/b200sv.h.  Nothing here is a translation of the reference kernels: index generation, vector widths,
// launch shapes and reductions are designed for H100 (128-bit accesses, 256-thread CTAs sized in multiples of
// the SM count, on-device final reductions with double atomics, no per-gate host synchronisation).
#include "sv_common.cuh"

#include <type_traits>

#include <math.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <mutex>

namespace b200sv {

static thread_local std::string g_err;
void set_error(const std::string& msg) { g_err = msg; }
int cuda_fail(cudaError_t e, const char* what)
{
    g_err = std::string(what) + ": " + cudaGetErrorString(e);
    cudaGetLastError();
    return (e == cudaErrorMemoryAllocation) ? B200SV_ENOMEM : B200SV_ECUDA;
}
static int einval(const char* msg)
{
    g_err = msg;
    return B200SV_EINVAL;
}

int sm_count(int dev)
{
    static std::mutex mtx;
    static std::map<int, int> cache;
    std::lock_guard<std::mutex> lk(mtx);
    auto it = cache.find(dev);
    if (it != cache.end()) {
        return it->second;
    }
    int n = 132; // H100 SXM; replaced by the queried value below
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    cache[dev] = n;
    return n;
}

// grid for a streaming kernel: enough CTAs for `items` one-per-thread, capped at 16 CTAs/SM (grid-stride beyond)
static inline unsigned stream_grid(int dev, uint64_t items, int block)
{
    const uint64_t need = (items + block - 1) / block;
    const uint64_t cap = (uint64_t)sm_count(dev) * 16U;
    return (unsigned)std::max<uint64_t>(1, std::min(need, cap));
}

// ---------------------------------------------------------------------------------------------------------
// reductions helpers
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        v += __shfl_xor_sync(0xffffffffu, v, o);
    }
    return v;
}
// block-wide sum -> one double atomic per CTA
__device__ __forceinline__ void block_atomic_add(double v, double* out)
{
    __shared__ double sh[32];
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) {
        sh[w] = v;
    }
    __syncthreads();
    if (w == 0) {
        const int nw = (blockDim.x + 31) >> 5;
        v = (lane < nw) ? sh[lane] : 0.0;
        v = warp_sum(v);
        if (lane == 0) {
            atomicAdd(out, v);
        }
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------------------------
// K1 (unfused form): generic Apply2x2 for arbitrary (offset1, offset2, sorted powers)
//   V = amplitudes per vector access (fp32: 2 -> 128-bit when the lowest involved qubit is >= 1)
//   ILP = independent pairs in flight per thread
// ---------------------------------------------------------------------------------------------------------
template <typename R, int V> struct VecT;
template <> struct VecT<float, 1> {
    typedef float2 type;
};
template <> struct VecT<float, 2> {
    typedef float4 type;
};
template <> struct VecT<double, 1> {
    typedef double2 type;
};

template <typename R, int V, bool NORM, int ILP>
__global__ void __launch_bounds__(256) k_apply2x2(typename Cx<R>::type* __restrict__ psi, uint64_t items, uint64_t off1,
    uint64_t off2, Mat2<R> mt, PowList pw, R thresh, double* normOut)
{
    typedef typename Cx<R>::type C;
    typedef typename VecT<R, V>::type Vec;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    double acc = 0.0;
    for (uint64_t j0 = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j0 < items; j0 += stride * ILP) {
        Vec a[ILP], b[ILP];
        uint64_t ia[ILP];
#pragma unroll
        for (int u = 0; u < ILP; ++u) {
            const uint64_t j = j0 + (uint64_t)u * stride;
            if (j < items) {
                const uint64_t i = push_apart(j * V, pw);
                ia[u] = i;
                a[u] = *reinterpret_cast<const Vec*>(psi + i + off1);
                b[u] = *reinterpret_cast<const Vec*>(psi + i + off2);
            }
        }
#pragma unroll
        for (int u = 0; u < ILP; ++u) {
            const uint64_t j = j0 + (uint64_t)u * stride;
            if (j < items) {
                C* pa = reinterpret_cast<C*>(&a[u]);
                C* pb = reinterpret_cast<C*>(&b[u]);
#pragma unroll
                for (int v = 0; v < V; ++v) {
                    C na = cmad2(mt.m[0], pa[v], mt.m[1], pb[v]);
                    C nb = cmad2(mt.m[2], pa[v], mt.m[3], pb[v]);
                    if (NORM) {
                        R n0 = cnorm(na), n1 = cnorm(nb);
                        if (n0 < thresh) {
                            na = mk<R>(0, 0);
                        } else {
                            acc += (double)n0;
                        }
                        if (n1 < thresh) {
                            nb = mk<R>(0, 0);
                        } else {
                            acc += (double)n1;
                        }
                    }
                    pa[v] = na;
                    pb[v] = nb;
                }
                *reinterpret_cast<Vec*>(psi + ia[u] + off1) = a[u];
                *reinterpret_cast<Vec*>(psi + ia[u] + off2) = b[u];
            }
        }
    }
    if (NORM) {
        block_atomic_add(acc, normOut);
    }
}

template <typename R> static Mat2<R> make_mat(const double* m8, double nrm)
{
    Mat2<R> mt;
    for (int k = 0; k < 4; ++k) {
        mt.m[k] = mk<R>((R)(m8[2 * k] * nrm), (R)(m8[2 * k + 1] * nrm));
    }
    return mt;
}

template <typename R>
static int launch_apply2x2(State* s, uint64_t off1, uint64_t off2, const double* m8, int nb, const uint64_t* pows,
    double nrm, double thresh, double* normOutDev)
{
    typedef typename Cx<R>::type C;
    PowList pw;
    pw.n = nb;
    for (int k = 0; k < nb; ++k) {
        pw.low[k] = pows[k] - 1U;
    }
    // For fp32 R the matrix is rounded to fp32 BEFORE the nrm fold when nrm==1 (bit-identical inputs to the oracle).
    Mat2<R> mt = make_mat<R>(m8, nrm);
    const uint64_t nItems = s->dim() >> nb;
    const bool norm = normOutDev != nullptr;
    C* psi = (C*)s->amps;
    const bool vec2 = (sizeof(R) == 4) && (nb == 0 || pows[0] >= 2U) && (nItems >= 2U);
    if (vec2) {
        const uint64_t items = nItems / 2U;
        const unsigned grid = stream_grid(s->dev, (items + 3) / 4, 256);
        if (norm) {
            k_apply2x2<float, 2, true, 4><<<grid, 256, 0, s->stream>>>(
                (float2*)psi, items, off1, off2, *(Mat2<float>*)&mt, pw, (float)thresh, normOutDev);
        } else {
            k_apply2x2<float, 2, false, 4><<<grid, 256, 0, s->stream>>>(
                (float2*)psi, items, off1, off2, *(Mat2<float>*)&mt, pw, (float)thresh, normOutDev);
        }
    } else {
        const unsigned grid = stream_grid(s->dev, (nItems + 3) / 4, 256);
        if (norm) {
            k_apply2x2<R, 1, true, 4><<<grid, 256, 0, s->stream>>>(psi, nItems, off1, off2, mt, pw, (R)thresh, normOutDev);
        } else {
            k_apply2x2<R, 1, false, 4><<<grid, 256, 0, s->stream>>>(psi, nItems, off1, off2, mt, pw, (R)thresh, normOutDev);
        }
    }
    SV_CUDA(cudaGetLastError());
    s->stats.kernel_launches++;
    s->stats.single_launches++;
    s->stats.bytes_swept += 2ULL * (nItems * 2ULL) * s->amp_bytes();
    return B200SV_OK;
}


// ---------------------------------------------------------------------------------------------------------
// 128-bit streaming helpers for the elementwise sweeps and reductions: every global access is one 16-byte chunk
// (fp32: amplitudes 2j and 2j+1 as a float4, fp64: one double2), grid-stride, so a warp touches 512 contiguous bytes per
// instruction.  f(i, amp) is called once per amplitude; map_amps writes the returned amplitude back.
// ---------------------------------------------------------------------------------------------------------
template <typename R, typename F>
__device__ __forceinline__ void for_amps(const typename Cx<R>::type* __restrict__ psi, uint64_t n, F f)
{
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint64_t gid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (sizeof(R) == 4 && n >= 2) {
        const float4* p = reinterpret_cast<const float4*>(psi);
        const uint64_t m = n >> 1;
        for (uint64_t j = gid; j < m; j += stride) {
            const float4 v = p[j];
            typename Cx<R>::type a0, a1;
            a0.x = (R)v.x;
            a0.y = (R)v.y;
            a1.x = (R)v.z;
            a1.y = (R)v.w;
            f(2U * j, a0);
            f(2U * j + 1U, a1);
        }
    } else {
        for (uint64_t i = gid; i < n; i += stride) {
            f(i, psi[i]);
        }
    }
}
template <typename R, typename F> __device__ __forceinline__ void map_amps(typename Cx<R>::type* psi, uint64_t n, F f)
{
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint64_t gid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (sizeof(R) == 4 && n >= 2) {
        float4* p = reinterpret_cast<float4*>(psi);
        const uint64_t m = n >> 1;
        for (uint64_t j = gid; j < m; j += stride) {
            const float4 v = p[j];
            typename Cx<R>::type a0, a1;
            a0.x = (R)v.x;
            a0.y = (R)v.y;
            a1.x = (R)v.z;
            a1.y = (R)v.w;
            a0 = f(2U * j, a0);
            a1 = f(2U * j + 1U, a1);
            p[j] = make_float4((float)a0.x, (float)a0.y, (float)a1.x, (float)a1.y);
        }
    } else {
        for (uint64_t i = gid; i < n; i += stride) {
            psi[i] = f(i, psi[i]);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// elementwise sweeps
// ---------------------------------------------------------------------------------------------------------
template <typename R>
__global__ void __launch_bounds__(256) k_apply_m(typename Cx<R>::type* psi, uint64_t n, uint64_t mask, uint64_t result,
    typename Cx<R>::type nrm)
{
    typedef typename Cx<R>::type C;
    // the dropped part is only WRITTEN (zeros): 1.5 instead of 2 state sizes of traffic.  128-bit accesses: fp32 handles the
    // amplitude pair (2j, 2j+1) per chunk and loads it only if at least one of the two is kept.
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint64_t gid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (sizeof(R) == 4 && n >= 2) {
        float4* p = reinterpret_cast<float4*>(psi);
        for (uint64_t j = gid; j < (n >> 1); j += stride) {
            const bool k0 = ((2U * j) & mask) == result, k1 = ((2U * j + 1U) & mask) == result;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (k0 | k1) {
                const float4 w = p[j];
                if (k0) {
                    v.x = (float)nrm.x * w.x - (float)nrm.y * w.y;
                    v.y = (float)nrm.x * w.y + (float)nrm.y * w.x;
                }
                if (k1) {
                    v.z = (float)nrm.x * w.z - (float)nrm.y * w.w;
                    v.w = (float)nrm.x * w.w + (float)nrm.y * w.z;
                }
            }
            p[j] = v;
        }
        return;
    }
    for (uint64_t i = gid; i < n; i += stride) {
        if ((i & mask) == result) {
            psi[i] = cmul<C>(nrm, psi[i]);
        } else {
            psi[i] = mk<R>(0, 0);
        }
    }
}

template <typename R>
__global__ void __launch_bounds__(256) k_collapse_parity(typename Cx<R>::type* psi, uint64_t n, uint64_t mask, int result,
    double* out)
{
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    double acc = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        if ((__popcll(i & mask) & 1) == result) {
            acc += (double)cnorm(psi[i]);
        } else {
            psi[i] = mk<R>(0, 0);
        }
    }
    block_atomic_add(acc, out);
}

template <typename R>
__global__ void __launch_bounds__(256) k_xmask(typename Cx<R>::type* psi, uint64_t half, uint64_t topLow, uint64_t mask)
{
    typedef typename Cx<R>::type C;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < half; j += stride) {
        const uint64_t lo = j & topLow;
        const uint64_t i = ((j ^ lo) << 1) | lo; // top mask bit clear
        const C a = psi[i];
        const C b = psi[i ^ mask];
        psi[i] = b;
        psi[i ^ mask] = a;
    }
}

template <typename R>
__global__ void __launch_bounds__(256) k_phase_parity(typename Cx<R>::type* psi, uint64_t n, uint64_t mask, uint64_t cmask,
    typename Cx<R>::type odd, typename Cx<R>::type even)
{
    typedef typename Cx<R>::type C;
    map_amps<R>(psi, n, [&](uint64_t i, C a) {
        if ((i & cmask) != cmask) {
            return a;
        }
        const bool p = __popcll(i & mask) & 1;
        return cmul<C>(p ? odd : even, a);
    });
}

template <typename R>
__global__ void __launch_bounds__(256) k_phase_root_n(typename Cx<R>::type* psi, uint64_t n, uint64_t mask, uint64_t nPhases,
    R radians)
{
    typedef typename Cx<R>::type C;
    map_amps<R>(psi, n, [&](uint64_t i, C a) {
        const uint64_t steps = (uint64_t)__popcll(i & mask) % nPhases;
        if (!steps) {
            return a;
        }
        R sn, cs;
        sincos(radians * (R)steps, &sn, &cs);
        return cmul<C>(mk<R>(cs, sn), a);
    });
}

template <typename R>
__global__ void __launch_bounds__(256) k_normalize(typename Cx<R>::type* psi, uint64_t n, typename Cx<R>::type f, R thresh)
{
    typedef typename Cx<R>::type C;
    map_amps<R>(psi, n, [&](uint64_t, C a) {
        if (cnorm(a) < thresh) {
            a = mk<R>(0, 0);
        }
        return cmul<C>(f, a);
    });
}

// UniformlyControlledSingleBit (reference state.cpp:1094-1198)
struct UcArgs {
    int nc;
    uint64_t cpow[32];
    int nskip;
    uint64_t skip[32];
    uint64_t skipValue;
};
template <typename R>
__global__ void __launch_bounds__(256) k_uniformly_controlled(typename Cx<R>::type* psi, uint64_t half, uint64_t tpow,
    const typename Cx<R>::type* __restrict__ mtrxs, UcArgs ua, R nrm)
{
    typedef typename Cx<R>::type C;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < half; j += stride) {
        const uint64_t lo = j & (tpow - 1U);
        const uint64_t i = ((j ^ lo) << 1) | lo;
        uint64_t off = 0;
        for (int c = 0; c < ua.nc; ++c) {
            if (i & ua.cpow[c]) {
                off |= 1ULL << c;
            }
        }
        uint64_t idx = 0, hi = off;
        for (int p = 0; p < ua.nskip; ++p) {
            const uint64_t l = hi & (ua.skip[p] - 1U);
            idx |= l;
            hi = (hi ^ l) << 1;
        }
        idx |= hi;
        const C* m = mtrxs + (idx | ua.skipValue) * 4U;
        const C a = psi[i], b = psi[i | tpow];
        C na = cmad2(m[0], a, m[1], b);
        C nb = cmad2(m[2], a, m[3], b);
        na.x *= nrm;
        na.y *= nrm;
        nb.x *= nrm;
        nb.y *= nrm;
        psi[i] = na;
        psi[i | tpow] = nb;
    }
}

// ---------------------------------------------------------------------------------------------------------
// reductions
// ---------------------------------------------------------------------------------------------------------
// All single-qubit marginals in ONE sweep: out[b] += sum of |psi_i|^2 over i with bit b set (b < nq), out[64] += total.
// Each thread walks groups of 8 consecutive amplitudes: bits 0..2 are resolved inside the group, every higher bit adds the
// group total once.  Accumulators are doubles in registers; one shuffle tree + one atomic per (block, bit) at the end.
template <typename R>
__global__ void __launch_bounds__(256) k_prob_all_bits(const typename Cx<R>::type* __restrict__ psi, uint64_t n, int nq, double* __restrict__ out)
{
    typedef typename Cx<R>::type C;
    double acc[40];
#pragma unroll
    for (int b = 0; b < 40; ++b) {
        acc[b] = 0.0;
    }
    double tot = 0.0;
    const uint64_t groups = n >> 3;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += stride) {
        const C* p = psi + (g << 3);
        R pr[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const C a = p[k];
            pr[k] = a.x * a.x + a.y * a.y;
        }
        const R s01 = pr[0] + pr[1], s23 = pr[2] + pr[3], s45 = pr[4] + pr[5], s67 = pr[6] + pr[7];
        const double gsum = (double)((s01 + s23) + (s45 + s67));
        tot += gsum;
        acc[0] += (double)((pr[1] + pr[3]) + (pr[5] + pr[7]));
        acc[1] += (double)(s23 + s67);
        acc[2] += (double)(s45 + s67);
#pragma unroll
        for (int b = 3; b < 40; ++b) {
            if (b < nq && ((g >> (b - 3)) & 1U)) {
                acc[b] += gsum;
            }
        }
    }
    __shared__ double red[8][41];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int b = 0; b < 41; ++b) {
        double v = (b < 40) ? acc[b < 40 ? b : 0] : tot;
        if (b < 40 && b >= nq) {
            continue;
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            v += __shfl_xor_sync(0xffffffffU, v, d);
        }
        if (lane == 0) {
            red[warp][b] = v;
        }
    }
    __syncthreads();
    const int b = threadIdx.x;
    if (b < 41 && (b == 40 || b < nq)) {
        double v = 0.0;
        for (int w = 0; w < 8; ++w) {
            v += red[w][b];
        }
        atomicAdd(out + (b == 40 ? 64 : b), v);
    }
}


// r2 version of the marginals sweep: coalesced 128-bit streaming loads and O(1) work per chunk.
// The state is 2^cl 16-byte chunks (fp32: amplitudes 2c, 2c+1; fp64: amplitude c).  Thread gid of a power-of-two grid reads
// chunk  it * T + gid  (T = total threads) for it = 0 .. 2^itBits - 1, so the chunk-index bits are, from the bottom: lane (5),
// warp (3), block (gBits), iteration (itBits).  Only the iteration bits vary inside a thread: their marginals come from a
// binary-counter (pairwise) summation — level b holds the sum of the last 2^b chunks with iteration bit b clear; when bit b
// is set the running value joins A[b] and absorbs the carry — amortised two float adds per chunk, uniform control flow across
// the whole grid (it depends on `it` only), and pairwise accuracy.  Lane / warp / block bits are resolved once at the end from
// the per-thread totals.  HBM traffic = one read of the state.
template <typename R, int MAXB>
__global__ void __launch_bounds__(256) k_prob_all_bits2(const typename Cx<R>::type* __restrict__ psi, int itBits, int gBits, int nq,
    double* __restrict__ out)
{
    constexpr int APCLOG = (sizeof(R) == 4) ? 1 : 0;
    const uint32_t tid = threadIdx.x;
    const uint64_t gid = (uint64_t)blockIdx.x * 256U + tid;
    const uint64_t T = (uint64_t)256U << gBits;
    const uint4* base = reinterpret_cast<const uint4*>(psi);
    typedef typename std::conditional<sizeof(R) == 4, float, double>::type Acc; // fp64 states keep their 1e-12 parity bar
    Acc A[MAXB], carry[MAXB];
#pragma unroll
    for (int b = 0; b < MAXB; ++b) {
        A[b] = 0;
        carry[b] = 0;
    }
    Acc a0 = 0, total = 0;
    // four independent 16-byte loads in flight per thread; the four chunk values are combined pairwise in registers (levels 0
    // and 1 of the counter), so the counter proper runs once per four chunks, starting at level 2
    const uint32_t nIt = 1U << itBits; // >= 4
    for (uint32_t it0 = 0; it0 < nIt; it0 += 4) {
        uint4 c[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            c[u] = __ldcs(base + ((uint64_t)(it0 + (uint32_t)u) * T + gid));
        }
        Acc w[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            if (APCLOG) {
                const float x0 = __uint_as_float(c[u].x), y0 = __uint_as_float(c[u].y), x1 = __uint_as_float(c[u].z), y1 = __uint_as_float(c[u].w);
                const float p1 = x1 * x1 + y1 * y1;
                a0 += (Acc)p1;
                w[u] = (Acc)((x0 * x0 + y0 * y0) + p1);
            } else {
                const double x = __hiloint2double((int)c[u].y, (int)c[u].x), y = __hiloint2double((int)c[u].w, (int)c[u].z);
                w[u] = (Acc)(x * x + y * y);
            }
        }
        A[0] += w[1] + w[3];
        const Acc w23 = w[2] + w[3];
        A[1] += w23;
        Acc v = (w[0] + w[1]) + w23;
        const uint32_t it = it0 >> 2;
        bool done = false;
#pragma unroll
        for (int b = 2; b < MAXB; ++b) {
            if (b < itBits && !done) {
                if ((it >> (b - 2)) & 1U) {
                    A[b] += v;
                    v += carry[b];
                } else {
                    carry[b] = v;
                    done = true;
                }
            }
        }
        if (!done) {
            total = v; // the last group: every level has been folded in
        }
    }
    // ---- per-thread results -> marginals.  Values reduced over the CTA: [0] total, [1] a0, [2 .. 2+itBits) A[b],
    // [2+MAXB .. +5) lane-bit sums, then warp-bit sums are formed from the per-warp totals.
    __shared__ double red[8][2 + MAXB + 5];
    const int lane = tid & 31, warp = tid >> 5;
    auto wsum = [](double v) {
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            v += __shfl_xor_sync(0xffffffffU, v, d);
        }
        return v;
    };
    {
        const double t = wsum((double)total), z = wsum((double)a0);
        if (lane == 0) {
            red[warp][0] = t;
            red[warp][1] = z;
        }
#pragma unroll
        for (int b = 0; b < MAXB; ++b) {
            if (b < itBits) {
                const double v = wsum((double)A[b]);
                if (lane == 0) {
                    red[warp][2 + b] = v;
                }
            }
        }
#pragma unroll
        for (int d = 0; d < 5; ++d) {
            const double v = wsum(((lane >> d) & 1) ? (double)total : 0.0);
            if (lane == 0) {
                red[warp][2 + MAXB + d] = v;
            }
        }
    }
    __syncthreads();
    const int j = (int)tid;
    if (j < 2 + MAXB + 5 + 3) {
        double v = 0.0;
        int qubit = -1; // -1: nothing, 64: total
        if (j < 2 + MAXB + 5) {
            for (int w = 0; w < 8; ++w) {
                v += red[w][j];
            }
            if (j == 0) {
                qubit = 64;
            } else if (j == 1) {
                qubit = APCLOG ? 0 : -1;
            } else if (j < 2 + MAXB) {
                qubit = (j - 2 < itBits) ? (APCLOG + 8 + gBits + (j - 2)) : -1;
            } else {
                qubit = APCLOG + (j - 2 - MAXB);
            }
        } else {
            const int wb = j - (2 + MAXB + 5); // warp bit
            for (int w = 0; w < 8; ++w) {
                if ((w >> wb) & 1) {
                    v += red[w][0];
                }
            }
            qubit = APCLOG + 5 + wb;
        }
        if (qubit >= 0 && (qubit == 64 || qubit < nq)) {
            atomicAdd(out + qubit, v);
        }
        if (j == 0) {
            // block bits: this CTA's total counts for every block-index bit that is set
            for (int g = 0; g < gBits; ++g) {
                if ((blockIdx.x >> g) & 1U) {
                    atomicAdd(out + (APCLOG + 8 + g), v);
                }
            }
        }
    }
}

template <typename R>
__global__ void __launch_bounds__(256) k_prob_mask(const typename Cx<R>::type* __restrict__ psi, uint64_t n, uint64_t mask,
    uint64_t perm, double* out)
{
    typedef typename Cx<R>::type C;
    double acc = 0;
    R part = 0;
    int cnt = 0;
    for_amps<R>(psi, n, [&](uint64_t i, C a) {
        if ((i & mask) == perm) {
            part += cnorm(a);
        }
        if (++cnt == 64) {
            acc += (double)part;
            part = 0;
            cnt = 0;
        }
    });
    acc += (double)part;
    block_atomic_add(acc, out);
}

// subset form: only the matching amplitudes are read (mask bits all >= 2^lowBit): j enumerates the free bits
template <typename R>
__global__ void __launch_bounds__(256) k_prob_mask_subset(const typename Cx<R>::type* __restrict__ psi, uint64_t items,
    PowList pw, uint64_t perm, double* out)
{
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    double acc = 0;
    R part = 0;
    int cnt = 0;
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < items; j += stride) {
        part += cnorm(psi[push_apart(j, pw) | perm]);
        if (++cnt == 64) {
            acc += (double)part;
            part = 0;
            cnt = 0;
        }
    }
    acc += (double)part;
    block_atomic_add(acc, out);
}

template <typename R>
__global__ void __launch_bounds__(256) k_prob_parity(const typename Cx<R>::type* __restrict__ psi, uint64_t n, uint64_t mask,
    double* out)
{
    typedef typename Cx<R>::type C;
    double acc = 0;
    R part = 0;
    int cnt = 0;
    for_amps<R>(psi, n, [&](uint64_t i, C a) {
        if (__popcll(i & mask) & 1) {
            part += cnorm(a);
        }
        if (++cnt == 64) {
            acc += (double)part;
            part = 0;
            cnt = 0;
        }
    });
    acc += (double)part;
    block_atomic_add(acc, out);
}

template <typename R>
__global__ void __launch_bounds__(256) k_norm(const typename Cx<R>::type* __restrict__ psi, uint64_t n, R thresh, double* out)
{
    typedef typename Cx<R>::type C;
    double acc = 0;
    R part = 0;
    int cnt = 0;
    for_amps<R>(psi, n, [&](uint64_t, C a) {
        const R v = cnorm(a);
        if (v >= thresh) {
            part += v;
        }
        if (++cnt == 64) {
            acc += (double)part;
            part = 0;
            cnt = 0;
        }
    });
    acc += (double)part;
    block_atomic_add(acc, out);
}

template <typename R>
__global__ void __launch_bounds__(256) k_inner(const typename Cx<R>::type* __restrict__ a, const typename Cx<R>::type* __restrict__ b,
    uint64_t n, double* out)
{
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    double re = 0, im = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const auto x = a[i];
        const auto y = b[i];
        // conj(x) * y
        re += (double)x.x * y.x + (double)x.y * y.y;
        im += (double)x.x * y.y - (double)x.y * y.x;
    }
    block_atomic_add(re, out);
    block_atomic_add(im, out + 1);
}

template <typename R, typename RO>
__global__ void __launch_bounds__(256) k_probs(const typename Cx<R>::type* __restrict__ psi, uint64_t n, RO* out)
{
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        out[i] = (RO)cnorm(psi[i]);
    }
}

__device__ __forceinline__ uint64_t pext64(uint64_t x, uint64_t mask)
{
    uint64_t r = 0;
    int k = 0;
    while (mask) {
        const uint64_t b = mask & (~mask + 1);
        if (x & b) {
            r |= 1ULL << k;
        }
        ++k;
        mask ^= b;
    }
    return r;
}

template <typename R>
__global__ void __launch_bounds__(256) k_prob_mask_all(const typename Cx<R>::type* __restrict__ psi, uint64_t n, uint64_t mask,
    double* bins, int useShared, int nbins)
{
    extern __shared__ double shbins[];
    if (useShared) {
        for (int b = threadIdx.x; b < nbins; b += blockDim.x) {
            shbins[b] = 0;
        }
        __syncthreads();
    }
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const double v = (double)cnorm(psi[i]);
        if (v != 0.0) {
            const uint64_t b = pext64(i, mask);
            if (useShared) {
                atomicAdd(&shbins[b], v);
            } else {
                atomicAdd(&bins[b], v);
            }
        }
    }
    if (useShared) {
        __syncthreads();
        for (int b = threadIdx.x; b < nbins; b += blockDim.x) {
            if (shbins[b] != 0.0) {
                atomicAdd(&bins[b], shbins[b]);
            }
        }
    }
}

// per-chunk sums of |psi|^2 (only terms > eps) for sampling; one CTA per chunk
template <typename R>
__global__ void __launch_bounds__(256) k_chunk_sums(const typename Cx<R>::type* __restrict__ psi, uint64_t chunk, R eps,
    double* sums)
{
    const uint64_t base = (uint64_t)blockIdx.x * chunk;
    double acc = 0;
    if (sizeof(R) == 4 && chunk >= 2) { // 128-bit loads: two amplitudes per access
        const float4* p = reinterpret_cast<const float4*>(psi + base);
        for (uint64_t j = threadIdx.x; j < (chunk >> 1); j += blockDim.x) {
            const float4 q = p[j];
            const float v0 = q.x * q.x + q.y * q.y, v1 = q.z * q.z + q.w * q.w;
            acc += (double)((v0 > (float)eps ? v0 : 0.f) + (v1 > (float)eps ? v1 : 0.f));
        }
    } else {
        for (uint64_t i = threadIdx.x; i < chunk; i += blockDim.x) {
            const R v = cnorm(psi[base + i]);
            if (v > eps) {
                acc += (double)v;
            }
        }
    }
    sums[blockIdx.x] = 0;
    __syncthreads();
    block_atomic_add(acc, sums + blockIdx.x);
}

// argmax |psi|^2 : packed (value bits, index) via 2-step: per-block best to arrays
template <typename R>
__global__ void __launch_bounds__(256) k_argmax(const typename Cx<R>::type* __restrict__ psi, uint64_t n, double* bestVal,
    unsigned long long* bestIdx)
{
    __shared__ double sv[256];
    __shared__ unsigned long long si[256];
    typedef typename Cx<R>::type C;
    double bv = -1;
    unsigned long long bi = 0;
    for_amps<R>(psi, n, [&](uint64_t i, C a) {
        const double v = (double)cnorm(a);
        if (v > bv || (v == bv && i < bi)) {
            bv = v;
            bi = i;
        }
    });
    sv[threadIdx.x] = bv;
    si[threadIdx.x] = bi;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) {
            const double ov = sv[threadIdx.x + o];
            const unsigned long long oi = si[threadIdx.x + o];
            if (ov > sv[threadIdx.x] || (ov == sv[threadIdx.x] && oi < si[threadIdx.x])) {
                sv[threadIdx.x] = ov;
                si[threadIdx.x] = oi;
            }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        bestVal[blockIdx.x] = sv[0];
        bestIdx[blockIdx.x] = si[0];
    }
}

// ---------------------------------------------------------------------------------------------------------
// structure kernels: Compose / Decompose / Dispose
// ---------------------------------------------------------------------------------------------------------
template <typename R>
__global__ void __launch_bounds__(256) k_compose(typename Cx<R>::type* __restrict__ out, const typename Cx<R>::type* __restrict__ a,
    const typename Cx<R>::type* __restrict__ b, uint64_t n, uint64_t startMask, uint64_t midMask, uint64_t endMask, int start,
    int nb)
{
    typedef typename Cx<R>::type C;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    if (sizeof(R) == 4 && start >= 1) {
        // fp32, inserted register above qubit 0: amplitudes 2j and 2j+1 share the b factor and are adjacent in a: 128-bit accesses
        float4* o4 = reinterpret_cast<float4*>(out);
        for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < (n >> 1); j += stride) {
            const uint64_t l = j << 1;
            const float4 x = *reinterpret_cast<const float4*>(a + ((l & startMask) | ((l & endMask) >> nb)));
            const C y = b[(l & midMask) >> start];
            o4[j] = make_float4(x.x * (float)y.x - x.y * (float)y.y, x.x * (float)y.y + x.y * (float)y.x, x.z * (float)y.x - x.w * (float)y.y,
                x.z * (float)y.y + x.w * (float)y.x);
        }
        return;
    }
    for (uint64_t l = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; l < n; l += stride) {
        const C x = a[(l & startMask) | ((l & endMask) >> nb)];
        const C y = b[(l & midMask) >> start];
        out[l] = cmul<C>(x, y);
    }
}

template <typename R>
__global__ void __launch_bounds__(256) k_dispose_perm(typename Cx<R>::type* __restrict__ out,
    const typename Cx<R>::type* __restrict__ in, uint64_t n, uint64_t skipMask, int length, uint64_t disposedRes)
{
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    if (sizeof(R) == 4 && (skipMask & 1U) && n >= 2) {
        // fp32, disposed register above qubit 0: kept amplitudes 2j, 2j+1 are adjacent in the source too
        float4* o4 = reinterpret_cast<float4*>(out);
        for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < (n >> 1); j += stride) {
            const uint64_t h = j << 1, lo = h & skipMask;
            o4[j] = *reinterpret_cast<const float4*>(in + (lo | ((h ^ lo) << length) | disposedRes));
        }
        return;
    }
    for (uint64_t h = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += stride) {
        const uint64_t lo = h & skipMask;
        out[h] = in[lo | ((h ^ lo) << length) | disposedRes];
    }
}

// One pass over psi accumulating the four marginals of DecomposeDispose (reference state.cpp:1605-1675):
//   remProb[r] = sum_k |psi|^2, remAngle[r] = sum_k arg(psi)|psi|^2 (only |psi|^2 > floor)
//   partProb[k] = sum_r |psi|^2, partAngle[k] = sum_r arg(psi)|psi|^2 (only |psi|^2 > floor)
// Accumulation is in double with atomics (shared-memory bins for the part side when it is small).
template <typename R>
__global__ void __launch_bounds__(256) k_decompose_marginals(const typename Cx<R>::type* __restrict__ psi, uint64_t n, int start,
    int length, R floorv, double* remProb, double* remAngle, double* partProb, double* partAngle, int partShared)
{
    extern __shared__ double sh[];
    const uint64_t partPower = 1ULL << length;
    if (partShared) {
        for (uint64_t b = threadIdx.x; b < 2 * partPower; b += blockDim.x) {
            sh[b] = 0;
        }
        __syncthreads();
    }
    const uint64_t startMask = (1ULL << start) - 1U;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const auto amp = psi[i];
        const R nrm = cnorm(amp);
        const uint64_t k = (i >> start) & (partPower - 1U);
        const uint64_t r = (i & startMask) | ((i >> (start + length)) << start);
        const double dn = (double)nrm;
        double ang = 0;
        if (nrm > floorv) {
            ang = (double)atan2(amp.y, amp.x) * dn;
        }
        if (dn != 0.0) {
            atomicAdd(&remProb[r], dn);
            if (ang != 0.0) {
                atomicAdd(&remAngle[r], ang);
            }
            if (partProb) {
                if (partShared) {
                    atomicAdd(&sh[k], dn);
                    atomicAdd(&sh[partPower + k], ang);
                } else {
                    atomicAdd(&partProb[k], dn);
                    atomicAdd(&partAngle[k], ang);
                }
            }
        }
    }
    if (partShared && partProb) {
        __syncthreads();
        for (uint64_t b = threadIdx.x; b < partPower; b += blockDim.x) {
            if (sh[b] != 0.0) {
                atomicAdd(&partProb[b], sh[b]);
            }
            if (sh[partPower + b] != 0.0) {
                atomicAdd(&partAngle[b], sh[partPower + b]);
            }
        }
    }
}


// r2 single-pass form of the marginals for the usual case that ONE side of the split is small (<= 2^11 entries; QUnit
// decomposes a few qubits out of a big register, or keeps a few).  The thread owns one index `o` of the LARGE side and walks
// the small side `j`: its row sums never leave registers and the rebuilt amplitude sqrt(P) e^{i theta} (state.cpp:1677-1695)
// is written straight to the new state — no 2^n doubles of accumulators, no per-amplitude global atomics.  The small side is
// summed per warp with shuffles (all lanes are at the same j), then per CTA in shared-memory bins, then one atomic per bin
// and CTA.  HBM traffic = one read of the state + one write of the large side.
//   smallIsPart = 1: o = remainder index, j = part index;  0: o = part index, j = remainder index.
template <typename R>
__global__ void __launch_bounds__(256) k_decompose_onepass(const typename Cx<R>::type* __restrict__ psi, int start, int length, int nq,
    int smallIsPart, R floorv, typename Cx<R>::type* __restrict__ outLarge, double* smallProb, double* smallAngle, int needSmall)
{
    extern __shared__ double sh[];
    const uint64_t partPower = 1ULL << length, remPower = 1ULL << (nq - length);
    const uint64_t smallN = smallIsPart ? partPower : remPower, largeN = smallIsPart ? remPower : partPower;
    if (needSmall) {
        for (uint64_t b = threadIdx.x; b < 2 * smallN; b += blockDim.x) {
            sh[b] = 0;
        }
        __syncthreads();
    }
    const uint64_t startMask = (1ULL << start) - 1U;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const int lane = threadIdx.x & 31;
    // every lane of a warp runs the same number of iterations (largeN is a power of two >= 32 or the tail lanes idle with zeros)
    const uint64_t rounds = (largeN + stride - 1U) / stride;
    for (uint64_t it = 0; it < rounds; ++it) {
        const uint64_t o = it * stride + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
        const bool live = o < largeN;
        double P = 0, A = 0;
        for (uint64_t j = 0; j < smallN; ++j) {
            const uint64_t r = smallIsPart ? o : j, k = smallIsPart ? j : o;
            double dn = 0, ang = 0;
            if (live) {
                const uint64_t i = (r & startMask) | (k << start) | ((r >> start) << (start + length));
                const auto amp = psi[i];
                const R nrm = cnorm(amp);
                dn = (double)nrm;
                if (nrm > floorv) {
                    ang = (double)atan2(amp.y, amp.x) * dn;
                }
                P += dn;
                A += ang;
            }
            if (needSmall) {
                const double wp = warp_sum(dn), wa = warp_sum(ang);
                if (lane == 0 && wp != 0.0) {
                    atomicAdd(&sh[j], wp);
                    if (wa != 0.0) {
                        atomicAdd(&sh[smallN + j], wa);
                    }
                }
            }
        }
        if (live) {
            const R p = (R)P;
            R th = (R)A;
            if (p > floorv) {
                th = (R)(A / P);
            }
            const R mag = (R)sqrt((double)p);
            R sn, cs;
            sincos(th, &sn, &cs);
            outLarge[o] = mk<R>(mag * cs, mag * sn);
        }
    }
    if (needSmall) {
        __syncthreads();
        for (uint64_t b = threadIdx.x; b < smallN; b += blockDim.x) {
            if (sh[b] != 0.0) {
                atomicAdd(&smallProb[b], sh[b]);
            }
            if (sh[smallN + b] != 0.0) {
                atomicAdd(&smallAngle[b], sh[smallN + b]);
            }
        }
    }
}

template <typename R>
__global__ void __launch_bounds__(256) k_polar_rebuild(typename Cx<R>::type* out, uint64_t n, const double* prob, const double* angle,
    R floorv)
{
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const R p = (R)prob[i];
        R ang = (R)angle[i];
        if (p > floorv) {
            ang = (R)(angle[i] / prob[i]);
        }
        const R mag = (R)sqrt((double)p);
        R sn, cs;
        sincos(ang, &sn, &cs);
        out[i] = mk<R>(mag * cs, mag * sn);
    }
}

template <typename C> __global__ void __launch_bounds__(256) k_swap_ranges(C* a, C* b, uint64_t n)
{
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const C x = a[i];
        a[i] = b[i];
        b[i] = x;
    }
}

// K7: fused re-page over NVLink.  dst[r'][c'] = src[c] with r' = victim bits of c, c' = c with the victim bits := rank bits.
struct ScatterArgs {
    uint4* dst[8 * 32]; // up to 2^8 destination pages
    int k;
    int cb[8];          // victim chunk-bit positions
    uint64_t vmask;     // OR of the victim chunk bits
    uint64_t rankDep;   // this rank's bits deposited at the victim positions
};
__global__ void __launch_bounds__(256) k_exchange_scatter(const uint4* __restrict__ src, uint64_t nChunks, const ScatterArgs* __restrict__ ap)
{
    __shared__ ScatterArgs a;
    for (unsigned i = threadIdx.x; i < sizeof(ScatterArgs) / 4; i += blockDim.x) {
        reinterpret_cast<unsigned*>(&a)[i] = reinterpret_cast<const unsigned*>(ap)[i];
    }
    __syncthreads();
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t c0 = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; c0 < nChunks; c0 += stride * 4) {
        uint4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const uint64_t c = c0 + u * stride;
            if (c < nChunks) {
                v[u] = src[c];
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const uint64_t c = c0 + u * stride;
            if (c < nChunks) {
                unsigned r = 0;
                for (int b = 0; b < a.k; ++b) {
                    r |= (unsigned)((c >> a.cb[b]) & 1ULL) << b;
                }
                a.dst[r][(c & ~a.vmask) | a.rankDep] = v[u];
            }
        }
    }
}

// The same re-page seen from the receiving side (PullArgs, sv_common.cuh): chunk c of this rank's new page comes from the rank
// named by the victim bits of c.  Used when a pending pull is not followed by a fused sweep that could carry it.
struct GatherArgs {
    const uint4* src[8];
    int cb[3];
    int k;
    uint64_t vmask, rankDep; // in chunks
};
__global__ void __launch_bounds__(256) k_exchange_gather(uint4* __restrict__ out, uint64_t nChunks, const __grid_constant__ GatherArgs a)
{
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t c0 = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; c0 < nChunks; c0 += stride * 4) {
        uint4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const uint64_t c = c0 + u * stride;
            if (c < nChunks) {
                unsigned r = 0;
                for (int b = 0; b < a.k; ++b) {
                    r |= (unsigned)((c >> a.cb[b]) & 1ULL) << b;
                }
                v[u] = a.src[r][(c & ~a.vmask) | a.rankDep];
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const uint64_t c = c0 + u * stride;
            if (c < nChunks) {
                out[c] = v[u];
            }
        }
    }
}

__global__ void k_fill_bytes(uint4* p, uint64_t n, unsigned v)
{
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        p[i] = make_uint4(v, v, v, v);
    }
}

// ---------------------------------------------------------------------------------------------------------
// host-side helpers
// ---------------------------------------------------------------------------------------------------------
struct DevGuard {
    int prev = -1;
    explicit DevGuard(int dev)
    {
        cudaGetDevice(&prev);
        if (prev != dev) {
            cudaSetDevice(dev);
        }
    }
    ~DevGuard()
    {
        int cur = -1;
        cudaGetDevice(&cur);
        if (prev >= 0 && cur != prev) {
            cudaSetDevice(prev);
        }
    }
};

static int ensure_scratch(State* s, size_t doubles)
{
    if (s->scratch_doubles >= doubles) {
        return B200SV_OK;
    }
    if (s->d_scratch) {
        cudaFree(s->d_scratch);
        cudaFreeHost(s->h_scratch);
        s->d_scratch = nullptr;
        s->h_scratch = nullptr;
        s->scratch_doubles = 0;
    }
    const size_t want = std::max<size_t>(doubles, 4096);
    SV_CUDA(cudaMalloc(&s->d_scratch, want * sizeof(double)));
    SV_CUDA(cudaMallocHost(&s->h_scratch, want * sizeof(double)));
    s->scratch_doubles = want;
    return B200SV_OK;
}


// ---- state-buffer cache --------------------------------------------------------------------------------------------------
// Compose / Decompose / Dispose replace the state buffer by one of another size, and QUnit-style callers do that all the time.
// cudaMalloc + cudaFree of GiB-sized buffers cost milliseconds each and synchronise the device (more than a Compose kernel at
// 30 qubits), so released state buffers are kept per device and handed out again on an exact size match.
struct BufCache {
    std::mutex m;
    struct Ent {
        void* p;
        size_t bytes;
    };
    std::vector<Ent> ent[64];
    size_t held[64] = { 0 };
};
static BufCache& buf_cache()
{
    static BufCache c;
    return c;
}
static void buf_cache_flush(int dev)
{
    BufCache& c = buf_cache();
    std::vector<BufCache::Ent> drop;
    {
        std::lock_guard<std::mutex> lk(c.m);
        drop.swap(c.ent[dev & 63]);
        c.held[dev & 63] = 0;
    }
    for (const BufCache::Ent& e : drop) {
        cudaFree(e.p);
    }
}
// current device must be `dev`
static cudaError_t state_buf_alloc(int dev, size_t bytes, void** out)
{
    BufCache& c = buf_cache();
    {
        std::lock_guard<std::mutex> lk(c.m);
        std::vector<BufCache::Ent>& v = c.ent[dev & 63];
        for (size_t i = 0; i < v.size(); ++i) {
            if (v[i].bytes == bytes) {
                *out = v[i].p;
                c.held[dev & 63] -= bytes;
                v.erase(v.begin() + (long)i);
                return cudaSuccess;
            }
        }
    }
    cudaError_t e = cudaMalloc(out, bytes);
    if (e == cudaErrorMemoryAllocation) {
        cudaGetLastError();
        buf_cache_flush(dev);
        e = cudaMalloc(out, bytes);
    }
    return e;
}
// the caller has synchronised every stream that used the buffer
static void state_buf_free(int dev, void* p, size_t bytes)
{
    if (!p) {
        return;
    }
    BufCache& c = buf_cache();
    static const size_t cap = [] {
        const char* e = getenv("B200SV_BUF_CACHE_MB");
        return (size_t)(e ? atoll(e) : 49152) << 20; // default: at most 48 GiB of released buffers per device
    }();
    {
        std::lock_guard<std::mutex> lk(c.m);
        std::vector<BufCache::Ent>& v = c.ent[dev & 63];
        if (bytes >= ((size_t)1 << 16) && v.size() < 8 && c.held[dev & 63] + bytes <= cap) {
            v.push_back({ p, bytes });
            c.held[dev & 63] += bytes;
            return;
        }
    }
    cudaFree(p);
}

static int alloc_amps(State* s, bool clear)
{
    if (s->amps) {
        return B200SV_OK;
    }
    if (s->external) {
        return einval("external buffer was released; cannot re-allocate");
    }
    const size_t bytes = (size_t)s->dim() * s->amp_bytes();
    cudaError_t e = state_buf_alloc(s->dev, bytes, &s->amps);
    if (e != cudaSuccess) {
        s->amps = nullptr;
        return cuda_fail(e, "cudaMalloc(state)");
    }
    s->amps_bytes = bytes;
    if (clear) {
        SV_CUDA(cudaMemsetAsync(s->amps, 0, bytes, s->stream));
    }
    return B200SV_OK;
}

static void free_amps(State* s)
{
    if ((s->amps && !s->external) || s->spare) {
        cudaStreamSynchronize(s->stream);
    }
    if (s->amps && !s->external) {
        if (s->amps_bytes) {
            state_buf_free(s->dev, s->amps, s->amps_bytes);
        } else {
            cudaFree(s->amps);
        }
    }
    s->amps_bytes = 0;
    if (s->spare) {
        cudaFree(s->spare); // the ping-pong buffer goes with the state it was sized for
        s->spare = nullptr;
        s->spare_bytes = 0;
    }
    s->amps = nullptr;
}

// make stream `waiter` wait for everything queued so far on `other`
static int cross_wait(State* waiter, State* other)
{
    if (waiter->stream == other->stream) {
        return B200SV_OK;
    }
    DevGuard g(other->dev);
    SV_CUDA(cudaEventRecord(other->evx, other->stream));
    SV_CUDA(cudaStreamWaitEvent(waiter->stream, other->evx, 0));
    return B200SV_OK;
}

static int read_scratch(State* s, int count)
{
    SV_CUDA(cudaMemcpyAsync(s->h_scratch, s->d_scratch, count * sizeof(double), cudaMemcpyDeviceToHost, s->stream));
    SV_CUDA(cudaStreamSynchronize(s->stream));
    return B200SV_OK;
}

template <typename R>
static int launch_apply2x2(State* s, uint64_t off1, uint64_t off2, const double* m8, int nb, const uint64_t* pows, double nrm, double thresh,
    double* normOutDev);

// A queued gate back in its (offset1, offset2, powers) form on the generic kernel
static int run_gate_unfused(State* s, const GateOp& g)
{
    uint64_t pows[64];
    int nb = 0;
    const uint64_t pmask = g.cmask | (1ULL << g.target);
    for (uint64_t m = pmask; m; m &= m - 1U) {
        pows[nb++] = m & (~m + 1U);
    }
    const uint64_t off1 = g.cval, off2 = g.cval | (1ULL << g.target);
    return (s->prec == 32) ? launch_apply2x2<float>(s, off1, off2, g.m, nb, pows, 1.0, 0.0, nullptr)
                           : launch_apply2x2<double>(s, off1, off2, g.m, nb, pows, 1.0, 0.0, nullptr);
}

int launch_pull_gather(State* s)
{
    if (!s->pullPending) {
        return B200SV_OK;
    }
    const int apcLog = (s->prec == 32) ? 1 : 0;
    GatherArgs a;
    memset(&a, 0, sizeof(a));
    a.k = s->pull.k;
    for (int b = 0; b < a.k; ++b) {
        a.cb[b] = s->pull.vb[b] - apcLog;
    }
    for (int r = 0; r < (1 << a.k); ++r) {
        a.src[r] = (const uint4*)s->pull.peers[r];
    }
    a.vmask = s->pull.vmask >> apcLog;
    a.rankDep = s->pull.rankDep >> apcLog;
    const uint64_t nChunks = (s->dim() * s->amp_bytes()) / 16U;
    const unsigned grid = stream_grid(s->dev, (nChunks + 3) / 4, 256);
    k_exchange_gather<<<grid, 256, 0, s->stream>>>((uint4*)s->pull.out, nChunks, a);
    SV_CUDA(cudaGetLastError());
    s->amps = s->pull.out;
    s->pullPending = false;
    s->stats.kernel_launches++;
    return B200SV_OK;
}

// the queue (and a pending re-page) no longer matter: the caller overwrites the whole state
static void drop_pending(State* s)
{
    s->queue.clear();
    if (s->pullPending) {
        s->amps = s->pull.out;
        s->pullPending = false;
    }
}

static int flush_queue(State* s)
{
    if (s->queue.empty()) {
        return s->pullPending ? launch_pull_gather(s) : B200SV_OK;
    }
    // fused_flush consumes the queue.  If its planner / encoder gives up (ESTATE: "no progress", "does not fit") nothing has been
    // launched yet, so the gates are replayed one by one on the generic kernel instead of being dropped; a CUDA failure
    // (launch, allocation) leaves the state undefined and is reported.
    std::vector<GateOp> saved;
    const bool keep = s->queue.size() <= 8192;
    if (keep) {
        saved = s->queue;
    }
    const int rc = fused_flush(s);
    if (rc == B200SV_ESTATE && keep) {
        s->queue.clear();
        SV_TRY(launch_pull_gather(s)); // (no-op unless a re-page is still pending)
        for (const GateOp& g : saved) {
            SV_TRY(run_gate_unfused(s, g));
        }
        return B200SV_OK;
    }
    return rc;
}

} // namespace b200sv

#include "alu_kernels.cuh"
#include "observables.cuh"
#include "rdm.cuh"

using namespace b200sv;

// read-only entry: keeps the memoised marginals
#define SV_ENTER_RO(s)                                                                                                 \
    if (!(s)) {                                                                                                        \
        set_error("null state handle");                                                                                \
        return B200SV_EINVAL;                                                                                          \
    }                                                                                                                  \
    DevGuard guard__((s)->dev)
// default entry: anything that is not explicitly read-only invalidates the memoised marginals
#define SV_ENTER(s)                                                                                                    \
    SV_ENTER_RO(s);                                                                                                    \
    (s)->margValid = false

#define DISPATCH_PREC(s, expr32, expr64)                                                                               \
    if ((s)->prec == 32) {                                                                                             \
        typedef float R;                                                                                               \
        typedef float2 C;                                                                                              \
        (void)sizeof(R);                                                                                               \
        (void)sizeof(C);                                                                                               \
        expr32;                                                                                                        \
    } else {                                                                                                           \
        typedef double R;                                                                                              \
        typedef double2 C;                                                                                             \
        (void)sizeof(R);                                                                                               \
        (void)sizeof(C);                                                                                               \
        expr64;                                                                                                        \
    }

extern "C" {

int b200sv_abi_version(void) { return 1; }
const char* b200sv_last_error(void) { return g_err.c_str(); }

int b200sv_device_count(int* count)
{
    if (!count) {
        return einval("null out pointer");
    }
    SV_CUDA(cudaGetDeviceCount(count));
    return B200SV_OK;
}

int b200sv_device_info(int dev, uint64_t* total_bytes, uint64_t* free_bytes, int* sms)
{
    DevGuard g(dev);
    size_t f = 0, t = 0;
    SV_CUDA(cudaMemGetInfo(&f, &t));
    if (total_bytes) {
        *total_bytes = t;
    }
    if (free_bytes) {
        *free_bytes = f;
    }
    if (sms) {
        *sms = sm_count(dev);
    }
    return B200SV_OK;
}

int b200sv_can_access_peer(int dev, int peer, int* can)
{
    if (!can) {
        return einval("null out pointer");
    }
    if (dev == peer) {
        *can = 1;
        return B200SV_OK;
    }
    SV_CUDA(cudaDeviceCanAccessPeer(can, dev, peer));
    return B200SV_OK;
}

static int create_common(int device, int n_qubits, int precision, void* ext, b200sv_t* out)
{
    if (!out) {
        return einval("null out pointer");
    }
    if (n_qubits < 0 || n_qubits > 40) {
        return einval("qubit count out of range");
    }
    if (precision != 32 && precision != 64) {
        return einval("precision must be 32 or 64");
    }
    int ndev = 0;
    SV_CUDA(cudaGetDeviceCount(&ndev));
    if (device < 0) {
        device = 0;
    }
    if (device >= ndev) {
        return einval("device index out of range");
    }
    DevGuard g(device);
    b200sv_state* s = new b200sv_state();
    s->dev = device;
    s->nq = n_qubits;
    s->prec = precision;
    s->amps = ext;
    s->external = ext != nullptr;
    cudaError_t e = cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) {
        e = cudaEventCreate(&s->ev0);
    }
    if (e == cudaSuccess) {
        e = cudaEventCreate(&s->ev1);
    }
    if (e == cudaSuccess) {
        e = cudaEventCreateWithFlags(&s->evx, cudaEventDisableTiming);
    }
    if (e != cudaSuccess) {
        delete s;
        return cuda_fail(e, "stream/event creation");
    }
    int r = ensure_scratch(s, 4096);
    if (r != B200SV_OK) {
        delete s;
        return r;
    }
    *out = s;
    return B200SV_OK;
}

int b200sv_create(int device, int n_qubits, int precision, b200sv_t* out)
{
    return create_common(device, n_qubits, precision, nullptr, out);
}

int b200sv_create_external(int device, int n_qubits, int precision, void* device_ptr, b200sv_t* out)
{
    if (!device_ptr) {
        return einval("null device pointer");
    }
    return create_common(device, n_qubits, precision, device_ptr, out);
}

int b200sv_destroy(b200sv_t s)
{
    if (!s) {
        return B200SV_OK;
    }
    DevGuard g(s->dev);
    cudaStreamSynchronize(s->stream);
    fused_release(s);
    free_amps(s);
    if (s->d_scratch) {
        cudaFree(s->d_scratch);
    }
    if (s->h_scratch) {
        cudaFreeHost(s->h_scratch);
    }
    if (s->d_flush) {
        cudaFree(s->d_flush);
    }
    cudaEventDestroy(s->ev0);
    cudaEventDestroy(s->ev1);
    cudaEventDestroy(s->evx);
    if (s->ownStream) {
        cudaStreamDestroy(s->stream);
    }
    delete s;
    return B200SV_OK;
}

int b200sv_qubit_count(b200sv_t s, int* n)
{
    if (!s || !n) {
        return einval("null argument");
    }
    *n = s->nq;
    return B200SV_OK;
}
int b200sv_precision(b200sv_t s, int* p)
{
    if (!s || !p) {
        return einval("null argument");
    }
    *p = s->prec;
    return B200SV_OK;
}
int b200sv_device(b200sv_t s, int* d)
{
    if (!s || !d) {
        return einval("null argument");
    }
    *d = s->dev;
    return B200SV_OK;
}

int b200sv_rebind_external(b200sv_t s, void* device_ptr)
{
    SV_ENTER(s);
    if (!s->external || !device_ptr) {
        return einval("rebind_external: not an external-buffer state or null pointer");
    }
    SV_TRY(flush_queue(s));
    s->amps = device_ptr; // stream order is preserved: later work on this state is queued behind the flush
    return B200SV_OK;
}

int b200sv_alloc_page(int device, uint64_t bytes, void** ptr)
{
    if (!ptr) {
        return einval("null out pointer");
    }
    DevGuard g(device);
    cudaError_t e = cudaMalloc(ptr, bytes);
    if (e != cudaSuccess) {
        *ptr = nullptr;
        return cuda_fail(e, "cudaMalloc(page)");
    }
    return B200SV_OK;
}
int b200sv_free_page(int device, void* ptr)
{
    DevGuard g(device);
    SV_CUDA(cudaDeviceSynchronize());
    SV_CUDA(cudaFree(ptr));
    return B200SV_OK;
}
int b200sv_ipc_export(int device, void* ptr, unsigned char handle_out[64])
{
    DevGuard g(device);
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    cudaIpcMemHandle_t h;
    SV_CUDA(cudaIpcGetMemHandle(&h, ptr));
    memcpy(handle_out, &h, 64);
    return B200SV_OK;
}
int b200sv_ipc_import(int device, const unsigned char handle[64], void** ptr)
{
    DevGuard g(device);
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    SV_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return B200SV_OK;
}
int b200sv_ipc_release(int device, void* ptr)
{
    DevGuard g(device);
    SV_CUDA(cudaIpcCloseMemHandle(ptr));
    return B200SV_OK;
}

int b200sv_exchange_scatter(b200sv_t s, int k, const int* victim_bits, int rank, void* const* dst_pages)
{
    SV_ENTER(s);
    if (k < 1 || k > 8 || !victim_bits || !dst_pages || rank < 0 || rank >= (1 << k)) {
        return einval("exchange_scatter: bad arguments (1 <= k <= 8, 0 <= rank < 2^k)");
    }
    if (!s->amps) {
        return einval("exchange_scatter: zero state");
    }
    const int apcLog = (s->prec == 32) ? 1 : 0;
    ScatterArgs a;
    memset(&a, 0, sizeof(a));
    a.k = k;
    for (int b = 0; b < k; ++b) {
        const int cb = victim_bits[b] - apcLog;
        if (cb < 0 || victim_bits[b] >= s->nq) {
            return einval("exchange_scatter: victim qubit out of range (must be a local qubit above the 16-byte chunk)");
        }
        for (int b2 = 0; b2 < b; ++b2) {
            if (a.cb[b2] == cb) {
                return einval("exchange_scatter: duplicate victim qubit");
            }
        }
        a.cb[b] = cb;
        a.vmask |= 1ULL << cb;
        if ((rank >> b) & 1) {
            a.rankDep |= 1ULL << cb;
        }
    }
    for (int r = 0; r < (1 << k); ++r) {
        if (!dst_pages[r]) {
            return einval("exchange_scatter: null destination page");
        }
        a.dst[r] = (uint4*)dst_pages[r];
    }
    SV_TRY(flush_queue(s));
    // argument block: reuse the per-state scratch (device) via pinned staging
    SV_TRY(ensure_scratch(s, (sizeof(ScatterArgs) + 7) / 8 + 8));
    memcpy(s->h_scratch, &a, sizeof(a));
    SV_CUDA(cudaMemcpyAsync(s->d_scratch, s->h_scratch, sizeof(a), cudaMemcpyHostToDevice, s->stream));
    const uint64_t nChunks = (s->dim() * s->amp_bytes()) / 16U;
    const unsigned grid = stream_grid(s->dev, (nChunks + 3) / 4, 256);
    k_exchange_scatter<<<grid, 256, 0, s->stream>>>((const uint4*)s->amps, nChunks, (const ScatterArgs*)s->d_scratch);
    SV_CUDA(cudaGetLastError());
    // the pinned staging block must not be overwritten before the copy has run
    SV_CUDA(cudaEventRecord(s->evx, s->stream));
    SV_CUDA(cudaEventSynchronize(s->evx));
    s->stats.kernel_launches++;
    return B200SV_OK;
}

static int fill_pull_args(int nq, int prec, int k, const int* victim_bits, int rank, const void* const* src_pages, void* out_page,
    PullArgs* pa)
{
    if (k < 1 || k > 3 || !victim_bits || !src_pages || !out_page || rank < 0 || rank >= (1 << k)) {
        return einval("exchange_pull: bad arguments (1 <= k <= 3)");
    }
    const int apcLog = (prec == 32) ? 1 : 0;
    memset(pa, 0, sizeof(*pa));
    pa->k = k;
    for (int b = 0; b < k; ++b) {
        if (victim_bits[b] < apcLog || victim_bits[b] >= nq) {
            return einval("exchange_pull: victim qubit out of range (must be a local qubit above the 16-byte chunk)");
        }
        for (int b2 = 0; b2 < b; ++b2) {
            if (victim_bits[b2] == victim_bits[b]) {
                return einval("exchange_pull: duplicate victim qubit");
            }
        }
        pa->vb[b] = victim_bits[b];
        pa->vmask |= 1ULL << victim_bits[b];
        if ((rank >> b) & 1) {
            pa->rankDep |= 1ULL << victim_bits[b];
        }
    }
    for (int r = 0; r < (1 << k); ++r) {
        if (!src_pages[r]) {
            return einval("exchange_pull: null source page");
        }
        if (src_pages[r] == out_page) {
            return einval("exchange_pull: the out page must differ from every source page");
        }
        pa->peers[r] = src_pages[r];
    }
    pa->out = out_page;
    return B200SV_OK;
}

int b200sv_exchange_pull(b200sv_t s, int k, const int* victim_bits, int rank, void* const* src_pages, void* out_page)
{
    SV_ENTER(s);
    if (!s->external || !s->amps) {
        return einval("exchange_pull: needs a state over an external page");
    }
    PullArgs pa;
    SV_TRY(fill_pull_args(s->nq, s->prec, k, victim_bits, rank, src_pages, out_page, &pa));
    SV_TRY(flush_queue(s)); // everything queued so far belongs to the old layout (and resolves an earlier pending pull)
    s->pull = pa;
    s->pullPending = true;
    return B200SV_OK;
}

int b200sv_set_stream(b200sv_t s, void* stream, int adopt)
{
    SV_ENTER(s);
    SV_TRY(flush_queue(s));
    SV_CUDA(cudaStreamSynchronize(s->stream));
    if (s->ownStream) {
        cudaStreamDestroy(s->stream);
    }
    if (adopt) {
        s->stream = (cudaStream_t)stream;
        s->ownStream = false;
    } else {
        SV_CUDA(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking));
        s->ownStream = true;
    }
    return B200SV_OK;
}

int b200sv_flush(b200sv_t s)
{
    SV_ENTER_RO(s);
    return flush_queue(s);
}

int b200sv_finish(b200sv_t s)
{
    SV_ENTER_RO(s);
    SV_TRY(flush_queue(s));
    SV_CUDA(cudaStreamSynchronize(s->stream));
    return B200SV_OK;
}

int b200sv_set_fusion(b200sv_t s, int mode)
{
    SV_ENTER(s);
    SV_TRY(flush_queue(s));
    s->fusion = mode;
    return B200SV_OK;
}

int b200sv_device_ptr(b200sv_t s, void** ptr)
{
    SV_ENTER(s);
    if (!ptr) {
        return einval("null out pointer");
    }
    SV_TRY(flush_queue(s));
    *ptr = s->amps;
    return B200SV_OK;
}

int b200sv_clone(b200sv_t s, b200sv_t* out)
{
    SV_ENTER(s);
    SV_TRY(flush_queue(s));
    b200sv_t c = nullptr;
    SV_TRY(b200sv_create(s->dev, s->nq, s->prec, &c));
    c->fusion = s->fusion;
    if (s->amps) {
        int r = alloc_amps(c, false);
        if (r != B200SV_OK) {
            b200sv_destroy(c);
            return r;
        }
        cross_wait(c, s);
        cudaError_t e = cudaMemcpyAsync(c->amps, s->amps, (size_t)s->dim() * s->amp_bytes(), cudaMemcpyDeviceToDevice, c->stream);
        if (e != cudaSuccess) {
            b200sv_destroy(c);
            return cuda_fail(e, "clone copy");
        }
        cross_wait(s, c);
    }
    *out = c;
    return B200SV_OK;
}

int b200sv_set_device(b200sv_t s, int device)
{
    SV_ENTER(s);
    if (device < 0 || device == s->dev) {
        return B200SV_OK;
    }
    int ndev = 0;
    SV_CUDA(cudaGetDeviceCount(&ndev));
    if (device >= ndev) {
        return einval("device index out of range");
    }
    if (s->external) {
        return einval("cannot migrate an external buffer");
    }
    SV_TRY(flush_queue(s));
    SV_CUDA(cudaStreamSynchronize(s->stream));
    fused_release(s); // the sweep-program arena lives on the old device
    // build the new-device resources, then move the buffer with a peer copy
    b200sv_t n = nullptr;
    SV_TRY(b200sv_create(device, s->nq, s->prec, &n));
    if (s->amps) {
        int r;
        {
            DevGuard g2(device);
            r = alloc_amps(n, false);
            if (r == B200SV_OK) {
                cudaError_t e = cudaMemcpyPeerAsync(n->amps, device, s->amps, s->dev, (size_t)s->dim() * s->amp_bytes(), n->stream);
                if (e == cudaSuccess) {
                    e = cudaStreamSynchronize(n->stream);
                }
                if (e != cudaSuccess) {
                    r = cuda_fail(e, "peer copy");
                }
            }
        }
        if (r != B200SV_OK) {
            b200sv_destroy(n);
            return r;
        }
    }
    // swap guts
    free_amps(s);
    std::swap(s->amps, n->amps);
    std::swap(s->amps_bytes, n->amps_bytes);
    std::swap(s->stream, n->stream);
    std::swap(s->ownStream, n->ownStream);
    std::swap(s->d_scratch, n->d_scratch);
    std::swap(s->h_scratch, n->h_scratch);
    std::swap(s->scratch_doubles, n->scratch_doubles);
    std::swap(s->d_flush, n->d_flush);
    std::swap(s->flush_bytes, n->flush_bytes);
    std::swap(s->ev0, n->ev0);
    std::swap(s->ev1, n->ev1);
    std::swap(s->evx, n->evx);
    std::swap(s->dev, n->dev);
    b200sv_destroy(n);
    return B200SV_OK;
}

// ---- state I/O ----------------------------------------------------------------------------------------------------

int b200sv_set_permutation(b200sv_t s, uint64_t perm, double re, double im)
{
    SV_ENTER(s);
    if (perm >= s->dim()) {
        return einval("SetPermutation: permutation out of bounds");
    }
    drop_pending(s); // Dump(): pending gates are irrelevant (reference state.cpp:230)
    SV_TRY(alloc_amps(s, false));
    SV_CUDA(cudaMemsetAsync(s->amps, 0, (size_t)s->dim() * s->amp_bytes(), s->stream));
    if (s->prec == 32) {
        const float2 v = make_float2((float)re, (float)im);
        SV_CUDA(cudaMemcpyAsync((float2*)s->amps + perm, &v, sizeof(v), cudaMemcpyHostToDevice, s->stream));
        SV_CUDA(cudaStreamSynchronize(s->stream));
    } else {
        const double2 v = make_double2(re, im);
        SV_CUDA(cudaMemcpyAsync((double2*)s->amps + perm, &v, sizeof(v), cudaMemcpyHostToDevice, s->stream));
        SV_CUDA(cudaStreamSynchronize(s->stream));
    }
    return B200SV_OK;
}

int b200sv_zero(b200sv_t s)
{
    SV_ENTER(s);
    drop_pending(s);
    if (s->external) {
        if (s->amps) {
            SV_CUDA(cudaMemsetAsync(s->amps, 0, (size_t)s->dim() * s->amp_bytes(), s->stream));
        }
        return B200SV_OK;
    }
    free_amps(s);
    return B200SV_OK;
}

int b200sv_is_zero(b200sv_t s, int* z)
{
    if (!s || !z) {
        return einval("null argument");
    }
    *z = (s->amps == nullptr);
    return B200SV_OK;
}

int b200sv_set_state(b200sv_t s, const void* host)
{
    SV_ENTER(s);
    if (!host) {
        return einval("null host pointer");
    }
    drop_pending(s);
    SV_TRY(alloc_amps(s, false));
    SV_CUDA(cudaMemcpyAsync(s->amps, host, (size_t)s->dim() * s->amp_bytes(), cudaMemcpyHostToDevice, s->stream));
    SV_CUDA(cudaStreamSynchronize(s->stream));
    return B200SV_OK;
}

int b200sv_get_state(b200sv_t s, void* host)
{
    SV_ENTER_RO(s);
    if (!host) {
        return einval("null host pointer");
    }
    SV_TRY(flush_queue(s));
    const size_t bytes = (size_t)s->dim() * s->amp_bytes();
    if (!s->amps) {
        memset(host, 0, bytes);
        return B200SV_OK;
    }
    SV_CUDA(cudaMemcpyAsync(host, s->amps, bytes, cudaMemcpyDeviceToHost, s->stream));
    SV_CUDA(cudaStreamSynchronize(s->stream));
    return B200SV_OK;
}

int b200sv_get_probs(b200sv_t s, void* host)
{
    SV_ENTER_RO(s);
    if (!host) {
        return einval("null host pointer");
    }
    SV_TRY(flush_queue(s));
    const uint64_t n = s->dim();
    const size_t rbytes = (s->prec == 32) ? 4 : 8;
    if (!s->amps) {
        memset(host, 0, n * rbytes);
        return B200SV_OK;
    }
    void* tmp = nullptr;
    SV_CUDA(cudaMalloc(&tmp, n * rbytes));
    const unsigned grid = stream_grid(s->dev, n, 256);
    if (s->prec == 32) {
        k_probs<float, float><<<grid, 256, 0, s->stream>>>((const float2*)s->amps, n, (float*)tmp);
    } else {
        k_probs<double, double><<<grid, 256, 0, s->stream>>>((const double2*)s->amps, n, (double*)tmp);
    }
    s->stats.kernel_launches++;
    cudaError_t e = cudaMemcpyAsync(host, tmp, n * rbytes, cudaMemcpyDeviceToHost, s->stream);
    if (e == cudaSuccess) {
        e = cudaStreamSynchronize(s->stream);
    }
    cudaFree(tmp);
    if (e != cudaSuccess) {
        return cuda_fail(e, "get_probs");
    }
    return B200SV_OK;
}

static bool bad_range(uint64_t off, uint64_t len, uint64_t dim) { return off > dim || len > dim - off; }

int b200sv_get_page(b200sv_t s, void* host, uint64_t offset, uint64_t length)
{
    SV_ENTER(s);
    if (bad_range(offset, length, s->dim())) {
        return einval("GetAmplitudePage range is out-of-bounds");
    }
    SV_TRY(flush_queue(s));
    const size_t ab = s->amp_bytes();
    if (!s->amps) {
        memset(host, 0, length * ab);
        return B200SV_OK;
    }
    SV_CUDA(cudaMemcpyAsync(host, (char*)s->amps + offset * ab, length * ab, cudaMemcpyDeviceToHost, s->stream));
    SV_CUDA(cudaStreamSynchronize(s->stream));
    return B200SV_OK;
}

int b200sv_set_page(b200sv_t s, const void* host, uint64_t offset, uint64_t length)
{
    SV_ENTER(s);
    if (bad_range(offset, length, s->dim())) {
        return einval("SetAmplitudePage range is out-of-bounds");
    }
    SV_TRY(flush_queue(s));
    if (!s->amps) {
        SV_TRY(alloc_amps(s, true));
    }
    const size_t ab = s->amp_bytes();
    SV_CUDA(cudaMemcpyAsync((char*)s->amps + offset * ab, host, length * ab, cudaMemcpyHostToDevice, s->stream));
    SV_CUDA(cudaStreamSynchronize(s->stream));
    return B200SV_OK;
}

static int enable_peer(int dev, int peer)
{
    if (dev == peer) {
        return B200SV_OK;
    }
    int can = 0;
    cudaDeviceCanAccessPeer(&can, dev, peer);
    if (!can) {
        return B200SV_ESTATE;
    }
    DevGuard g(dev);
    cudaError_t e = cudaDeviceEnablePeerAccess(peer, 0);
    if (e == cudaErrorPeerAccessAlreadyEnabled) {
        cudaGetLastError();
        e = cudaSuccess;
    }
    return e == cudaSuccess ? B200SV_OK : B200SV_ESTATE;
}

int b200sv_copy_page(b200sv_t dst, b200sv_t src, uint64_t src_off, uint64_t dst_off, uint64_t length)
{
    SV_ENTER(dst);
    if (!src) {
        return einval("null source handle");
    }
    if (dst->prec != src->prec) {
        return einval("precision mismatch");
    }
    if (bad_range(dst_off, length, dst->dim()) || bad_range(src_off, length, src->dim())) {
        return einval("SetAmplitudePage source/destination range is out-of-bounds");
    }
    {
        DevGuard g2(src->dev);
        SV_TRY(flush_queue(src));
    }
    SV_TRY(flush_queue(dst));
    if (!dst->amps && !src->amps) {
        return B200SV_OK;
    }
    if (!src->amps && length == dst->dim()) {
        return b200sv_zero(dst);
    }
    if (!dst->amps) {
        SV_TRY(alloc_amps(dst, true));
    }
    const size_t ab = dst->amp_bytes();
    if (!src->amps) {
        SV_CUDA(cudaMemsetAsync((char*)dst->amps + dst_off * ab, 0, length * ab, dst->stream));
        return B200SV_OK;
    }
    SV_TRY(cross_wait(dst, src));
    if (dst->dev == src->dev) {
        SV_CUDA(cudaMemcpyAsync((char*)dst->amps + dst_off * ab, (char*)src->amps + src_off * ab, length * ab,
            cudaMemcpyDeviceToDevice, dst->stream));
    } else {
        enable_peer(dst->dev, src->dev);
        SV_CUDA(cudaMemcpyPeerAsync((char*)dst->amps + dst_off * ab, dst->dev, (char*)src->amps + src_off * ab, src->dev,
            length * ab, dst->stream));
    }
    SV_TRY(cross_wait(src, dst));
    return B200SV_OK;
}

int b200sv_shuffle(b200sv_t a, b200sv_t b)
{
    SV_ENTER(a);
    if (!b) {
        return einval("null handle");
    }
    b->margValid = false;
    if (a->nq != b->nq || a->prec != b->prec) {
        return einval("ShuffleBuffers argument size differs from this");
    }
    {
        DevGuard g2(b->dev);
        SV_TRY(flush_queue(b));
    }
    SV_TRY(flush_queue(a));
    if (!a->amps && !b->amps) {
        return B200SV_OK;
    }
    if (!a->amps) {
        SV_TRY(alloc_amps(a, true));
    }
    if (!b->amps) {
        DevGuard g2(b->dev);
        SV_TRY(alloc_amps(b, true));
    }
    const uint64_t half = a->dim() >> 1;
    const size_t ab = a->amp_bytes();
    SV_TRY(cross_wait(a, b));
    char* pa = (char*)a->amps + half * ab; // upper half of a
    char* pb = (char*)b->amps;             // lower half of b
    const bool direct = (a->dev == b->dev) || (enable_peer(a->dev, b->dev) == B200SV_OK);
    if (direct) {
        // one kernel on a's SMs reads and writes b's half through NVLink peer mapping.  16-byte words, except when half a
        // page is smaller than one (a 1-qubit fp32 state: one 8-byte amplitude, which is also not 16-byte aligned in a)
        if ((half * ab) % 16U) {
            const uint64_t n8 = half * ab / 8;
            k_swap_ranges<uint2><<<stream_grid(a->dev, n8, 256), 256, 0, a->stream>>>((uint2*)pa, (uint2*)pb, n8);
        } else {
            const uint64_t n16 = half * ab / 16;
            k_swap_ranges<uint4><<<stream_grid(a->dev, n16, 256), 256, 0, a->stream>>>((uint4*)pa, (uint4*)pb, n16);
        }
        SV_CUDA(cudaGetLastError());
        a->stats.kernel_launches++;
    } else {
        // no peer access between the two devices: staged through a buffer on a's device (from the state-buffer cache: a
        // QPager meta gate calls this twice per gate), every copy checked
        void* tmp = nullptr;
        cudaError_t e = state_buf_alloc(a->dev, half * ab, &tmp);
        if (e != cudaSuccess) {
            return cuda_fail(e, "cudaMalloc(shuffle staging)");
        }
        e = cudaMemcpyAsync(tmp, pa, half * ab, cudaMemcpyDeviceToDevice, a->stream);
        if (e == cudaSuccess) {
            e = cudaMemcpyPeerAsync(pa, a->dev, pb, b->dev, half * ab, a->stream);
        }
        if (e == cudaSuccess) {
            e = cudaMemcpyPeerAsync(pb, b->dev, tmp, a->dev, half * ab, a->stream);
        }
        const cudaError_t es = cudaStreamSynchronize(a->stream);
        state_buf_free(a->dev, tmp, half * ab);
        if (e != cudaSuccess || es != cudaSuccess) {
            return cuda_fail(e != cudaSuccess ? e : es, "shuffle (staged)");
        }
    }
    SV_TRY(cross_wait(b, a));
    return B200SV_OK;
}

int b200sv_copy_state(b200sv_t dst, b200sv_t src)
{
    if (!dst || !src) {
        return einval("null handle");
    }
    dst->margValid = false;
    if (dst->nq != src->nq) {
        return einval("CopyStateVec argument size differs from this");
    }
    if (!src->amps && src->queue.empty()) {
        return b200sv_zero(dst);
    }
    drop_pending(dst);
    return b200sv_copy_page(dst, src, 0, 0, src->dim());
}

int b200sv_get_amplitude(b200sv_t s, uint64_t perm, double* re, double* im)
{
    SV_ENTER_RO(s);
    if (perm >= s->dim()) {
        return einval("GetAmplitude argument out-of-bounds");
    }
    SV_TRY(flush_queue(s));
    if (!s->amps) {
        *re = 0;
        *im = 0;
        return B200SV_OK;
    }
    if (s->prec == 32) {
        float2 v;
        SV_CUDA(cudaMemcpyAsync(&v, (float2*)s->amps + perm, sizeof(v), cudaMemcpyDeviceToHost, s->stream));
        SV_CUDA(cudaStreamSynchronize(s->stream));
        *re = v.x;
        *im = v.y;
    } else {
        double2 v;
        SV_CUDA(cudaMemcpyAsync(&v, (double2*)s->amps + perm, sizeof(v), cudaMemcpyDeviceToHost, s->stream));
        SV_CUDA(cudaStreamSynchronize(s->stream));
        *re = v.x;
        *im = v.y;
    }
    return B200SV_OK;
}

int b200sv_set_amplitude(b200sv_t s, uint64_t perm, double re, double im)
{
    SV_ENTER(s);
    if (perm >= s->dim()) {
        return einval("SetAmplitude argument out-of-bounds");
    }
    SV_TRY(flush_queue(s));
    if (!s->amps) {
        if (re == 0.0 && im == 0.0) {
            return B200SV_OK;
        }
        SV_TRY(alloc_amps(s, true));
    }
    if (s->prec == 32) {
        const float2 v = make_float2((float)re, (float)im);
        SV_CUDA(cudaMemcpyAsync((float2*)s->amps + perm, &v, sizeof(v), cudaMemcpyHostToDevice, s->stream));
    } else {
        const double2 v = make_double2(re, im);
        SV_CUDA(cudaMemcpyAsync((double2*)s->amps + perm, &v, sizeof(v), cudaMemcpyHostToDevice, s->stream));
    }
    SV_CUDA(cudaStreamSynchronize(s->stream));
    return B200SV_OK;
}

// (offset1, offset2, powers) single-target form -> queued gate (shared by b200sv_apply2x2 and the emulation hook)
static void make_gate_op(int prec, uint64_t off1, uint64_t off2, uint64_t pmask, const double* m8, double nrm, GateOp& g)
{
    const uint64_t diff = off1 ^ off2;
    g.target = __builtin_ctzll(diff);
    g.cmask = pmask & ~diff;
    g.cval = off1 & ~diff;
    const bool swapped = (off1 & diff) != 0; // off1 holds the |1> branch: reorder the matrix
    const int ord[4] = { 3, 2, 1, 0 };
    for (int k = 0; k < 4; ++k) {
        const int src = swapped ? ord[k] : k;
        g.m[2 * k] = m8[2 * src] * nrm;
        g.m[2 * k + 1] = m8[2 * src + 1] * nrm;
    }
    if (prec == 32) {
        for (int k = 0; k < 8; ++k) {
            g.m[k] = (double)(float)g.m[k];
        }
    }
    const bool z1 = g.m[2] == 0 && g.m[3] == 0, z2 = g.m[4] == 0 && g.m[5] == 0;
    const bool z0 = g.m[0] == 0 && g.m[1] == 0, z3 = g.m[6] == 0 && g.m[7] == 0;
    g.kind = (z1 && z2) ? 1 : ((z0 && z3) ? 2 : 0);
}

// ---- gates -----------------------------------------------------------------------------------------------------------

int b200sv_apply2x2(b200sv_t s, uint64_t off1, uint64_t off2, const double* m8, int bit_count, const uint64_t* pows,
    double nrm, double norm_thresh, double* norm_out)
{
    SV_ENTER(s);
    if (!m8 || (bit_count > 0 && !pows)) {
        return einval("Apply2x2: null argument");
    }
    const uint64_t dim = s->dim();
    if (off1 >= dim || off2 >= dim) {
        return einval("Apply2x2 offset1 and offset2 parameters must be within allocated qubit bounds!");
    }
    if (bit_count < 0 || bit_count > s->nq) {
        return einval("Apply2x2: bad bit count");
    }
    uint64_t pmask = 0;
    for (int k = 0; k < bit_count; ++k) {
        if (pows[k] >= dim || !pows[k] || (pows[k] & (pows[k] - 1U))) {
            return einval("Apply2x2 parameter qPowsSorted array values must be within allocated qubit bounds!");
        }
        if (k && pows[k - 1] >= pows[k]) {
            return einval("Apply2x2 parameter qPowSorted array values must be sorted and cannot be duplicated!");
        }
        pmask |= pows[k];
    }
    if ((off1 & ~pmask) || (off2 & ~pmask)) {
        return einval("Apply2x2: offsets must be combinations of the given powers");
    }
    if (!s->amps) { // CHECK_ZERO_SKIP
        if (norm_out) {
            *norm_out = 0;
        }
        return B200SV_OK;
    }
    s->stats.gates_submitted++;
    // queue single-target gates for the fused sweep
    const uint64_t diff = off1 ^ off2;
    if (!norm_out && s->fusion && diff && !(diff & (diff - 1U))) {
        GateOp g;
        make_gate_op(s->prec, off1, off2, pmask, m8, nrm, g);
        if (fused_accepts(s, g)) {
            s->queue.push_back(g);
            if (s->queue.size() >= 4096) {
                SV_TRY(flush_queue(s));
            }
            return B200SV_OK;
        }
    }
    SV_TRY(flush_queue(s));
    double* dn = nullptr;
    if (norm_out) {
        dn = s->d_scratch;
        SV_CUDA(cudaMemsetAsync(dn, 0, sizeof(double), s->stream));
    }
    if (s->prec == 32) {
        SV_TRY(launch_apply2x2<float>(s, off1, off2, m8, bit_count, pows, nrm, norm_thresh, dn));
    } else {
        SV_TRY(launch_apply2x2<double>(s, off1, off2, m8, bit_count, pows, nrm, norm_thresh, dn));
    }
    if (norm_out) {
        SV_TRY(read_scratch(s, 1));
        *norm_out = s->h_scratch[0];
    }
    return B200SV_OK;
}

int b200sv_apply_gates(b200sv_t s, int n_gates, const uint64_t* off1, const uint64_t* off2, const uint64_t* pmasks, const double* mats8)
{
    SV_ENTER(s);
    if (n_gates < 0 || (n_gates && (!off1 || !off2 || !pmasks || !mats8))) {
        return einval("apply_gates: null argument");
    }
    for (int i = 0; i < n_gates; ++i) {
        const uint64_t diff = off1[i] ^ off2[i];
        if (!diff || (diff & (diff - 1U)) || (pmasks[i] >> s->nq) || ((off1[i] | off2[i]) & ~pmasks[i])) {
            return einval("apply_gates: every gate must be a single-target Apply2x2 form within the qubit bounds");
        }
    }
    if (!s->amps) { // CHECK_ZERO_SKIP
        return B200SV_OK;
    }
    for (int i = 0; i < n_gates; ++i) {
        GateOp g;
        make_gate_op(s->prec, off1[i], off2[i], pmasks[i], mats8 + 8 * (size_t)i, 1.0, g);
        s->stats.gates_submitted++;
        if (s->fusion && fused_accepts(s, g)) {
            s->queue.push_back(g);
            if (s->queue.size() >= 4096) {
                SV_TRY(flush_queue(s));
            }
            continue;
        }
        // unfused engines (tiny registers, fusion switched off): the generic kernel, gate by gate
        SV_TRY(flush_queue(s));
        SV_TRY(run_gate_unfused(s, g));
    }
    return B200SV_OK;
}

int b200sv_xmask(b200sv_t s, uint64_t mask)
{
    SV_ENTER(s);
    if (mask >= s->dim()) {
        return einval("XMask mask out-of-bounds!");
    }
    if (!s->amps || !mask) {
        return B200SV_OK;
    }
    if (s->fusion && s->nq >= 5) {
        // queued as X gates: the fused scheduler turns the XMask ... XMask wrappers of anti-controlled gates
        // (QInterface::MACWrapper, include/qinterface.hpp:179-189) into control polarities, and hands a wide XMask that
        // nothing absorbed back to launch_xmask at flush time
        static const double xm[8] = { 0, 0, 1, 0, 1, 0, 0, 0 };
        for (uint64_t m = mask; m; m &= m - 1U) {
            GateOp g;
            const uint64_t p = m & (~m + 1U);
            make_gate_op(s->prec, 0, p, p, xm, 1.0, g);
            s->queue.push_back(g);
        }
        s->stats.gates_submitted++;
        if (s->queue.size() >= 4096) {
            SV_TRY(flush_queue(s));
        }
        return B200SV_OK;
    }
    SV_TRY(flush_queue(s));
    return launch_xmask(s, mask);
}
} // extern "C"

int b200sv::launch_xmask(State* s, uint64_t mask)
{
    const uint64_t half = s->dim() >> 1;
    const uint64_t top = 1ULL << (63 - __builtin_clzll(mask));
    const unsigned grid = stream_grid(s->dev, half, 256);
    DISPATCH_PREC(s, (k_xmask<float><<<grid, 256, 0, s->stream>>>((float2*)s->amps, half, top - 1U, mask)),
        (k_xmask<double><<<grid, 256, 0, s->stream>>>((double2*)s->amps, half, top - 1U, mask)));
    SV_CUDA(cudaGetLastError());
    s->stats.kernel_launches++;
    return B200SV_OK;
}

extern "C" {

int b200sv_phase_parity(b200sv_t s, double radians, uint64_t mask)
{
    SV_ENTER(s);
    if (mask >= s->dim()) {
        return einval("PhaseParity mask out-of-bounds!");
    }
    if (!s->amps || !mask) {
        return B200SV_OK;
    }
    SV_TRY(flush_queue(s));
    const uint64_t n = s->dim();
    const unsigned grid = stream_grid(s->dev, n, 256);
    if (s->prec == 32) {
        const float ang = (float)(radians / 2);
        const float cs = (float)cos(ang), sn = (float)sin(ang);
        k_phase_parity<float><<<grid, 256, 0, s->stream>>>((float2*)s->amps, n, mask, 0, make_float2(cs, sn), make_float2(cs, -sn));
    } else {
        const double ang = radians / 2;
        const double cs = cos(ang), sn = sin(ang);
        k_phase_parity<double><<<grid, 256, 0, s->stream>>>((double2*)s->amps, n, mask, 0, make_double2(cs, sn), make_double2(cs, -sn));
    }
    SV_CUDA(cudaGetLastError());
    s->stats.kernel_launches++;
    return B200SV_OK;
}

int b200sv_uniform_parity_rz(b200sv_t s, uint64_t control_mask, uint64_t mask, double angle)
{
    SV_ENTER(s);
    if (mask >= s->dim() || control_mask >= s->dim()) {
        return einval("UniformParityRZ mask out-of-bounds!");
    }
    if (!s->amps) {
        return B200SV_OK;
    }
    SV_TRY(flush_queue(s));
    const uint64_t n = s->dim();
    const unsigned grid = stream_grid(s->dev, n, 256);
    if (s->prec == 32) {
        const float cs = (float)cos(angle), sn = (float)sin(angle);
        k_phase_parity<float><<<grid, 256, 0, s->stream>>>((float2*)s->amps, n, mask, control_mask, make_float2(cs, sn), make_float2(cs, -sn));
    } else {
        const double cs = cos(angle), sn = sin(angle);
        k_phase_parity<double><<<grid, 256, 0, s->stream>>>((double2*)s->amps, n, mask, control_mask, make_double2(cs, sn), make_double2(cs, -sn));
    }
    SV_CUDA(cudaGetLastError());
    s->stats.kernel_launches++;
    return B200SV_OK;
}

int b200sv_phase_root_n_mask(b200sv_t s, int n, uint64_t mask)
{
    SV_ENTER(s);
    if (mask >= s->dim()) {
        return einval("PhaseRootNMask mask out-of-bounds!");
    }
    if (!s->amps || !n || !mask) {
        return B200SV_OK;
    }
    SV_TRY(flush_queue(s));
    const uint64_t dim = s->dim();
    const unsigned grid = stream_grid(s->dev, dim, 256);
    const uint64_t nPhases = 1ULL << n;
    if (s->prec == 32) {
        const float radians = (float)(-(double)(float)M_PI / (double)(1ULL << (n - 1)));
        k_phase_root_n<float><<<grid, 256, 0, s->stream>>>((float2*)s->amps, dim, mask, nPhases, radians);
    } else {
        const double radians = -M_PI / (double)(1ULL << (n - 1));
        k_phase_root_n<double><<<grid, 256, 0, s->stream>>>((double2*)s->amps, dim, mask, nPhases, radians);
    }
    SV_CUDA(cudaGetLastError());
    s->stats.kernel_launches++;
    return B200SV_OK;
}

int b200sv_uniformly_controlled(b200sv_t s, int n_controls, const int* controls, int target, const double* mtrxs, int n_skip,
    const uint64_t* skip_powers, uint64_t skip_value_mask, double nrm)
{
    SV_ENTER(s);
    // the matrix table holds 2^(n_controls + n_skip) 2x2 matrices: bounded so that its size cannot overflow, and every index
    // the kernel forms (control bits with zeros inserted at the skip powers, OR the skip value mask) stays inside it
    if (target < 0 || target >= s->nq || n_controls < 0 || n_skip < 0 || n_controls > 30 || n_skip > 30 - n_controls) {
        return einval("UniformlyControlledSingleBit argument out-of-bounds!");
    }
    if (!mtrxs || (n_controls && !controls) || (n_skip && !skip_powers)) {
        return einval("UniformlyControlledSingleBit: null array argument");
    }
    for (int c = 0; c < n_controls; ++c) {
        if (controls[c] < 0 || controls[c] >= s->nq) {
            return einval("UniformlyControlledSingleBit control is out-of-bounds!");
        }
    }
    const uint64_t tableSize = 1ULL << (n_controls + n_skip);
    for (int c = 0; c < n_skip; ++c) {
        if (!skip_powers[c] || (skip_powers[c] & (skip_powers[c] - 1U)) || skip_powers[c] >= tableSize) {
            return einval("UniformlyControlledSingleBit skip power is not a power of two inside the matrix table!");
        }
    }
    if (skip_value_mask >= tableSize) {
        return einval("UniformlyControlledSingleBit skip value mask is outside the matrix table!");
    }
    if (!s->amps) {
        return B200SV_OK;
    }
    SV_TRY(flush_queue(s));
    UcArgs ua;
    ua.nc = n_controls;
    for (int c = 0; c < n_controls; ++c) {
        ua.cpow[c] = 1ULL << controls[c];
    }
    ua.nskip = n_skip;
    for (int c = 0; c < n_skip; ++c) {
        ua.skip[c] = skip_powers[c];
    }
    ua.skipValue = skip_value_mask;
    const size_t nm = (size_t)tableSize * 4U;
    const uint64_t half = s->dim() >> 1;
    const unsigned grid = stream_grid(s->dev, half, 256);
    void* dm = nullptr;
    if (s->prec == 32) {
        std::vector<float2> hm;
        try {
            hm.resize(nm);
        } catch (const std::bad_alloc&) {
            set_error("UniformlyControlledSingleBit: host memory for the fp32 matrix table");
            return B200SV_ENOMEM;
        }
        for (size_t k = 0; k < nm; ++k) {
            hm[k] = make_float2((float)mtrxs[2 * k], (float)mtrxs[2 * k + 1]);
        }
        SV_CUDA(cudaMalloc(&dm, nm * sizeof(float2)));
        cudaMemcpyAsync(dm, hm.data(), nm * sizeof(float2), cudaMemcpyHostToDevice, s->stream);
        cudaStreamSynchronize(s->stream);
        k_uniformly_controlled<float><<<grid, 256, 0, s->stream>>>((float2*)s->amps, half, 1ULL << target, (const float2*)dm, ua, (float)nrm);
    } else {
        SV_CUDA(cudaMalloc(&dm, nm * sizeof(double2)));
        cudaMemcpyAsync(dm, mtrxs, nm * sizeof(double2), cudaMemcpyHostToDevice, s->stream);
        cudaStreamSynchronize(s->stream);
        k_uniformly_controlled<double><<<grid, 256, 0, s->stream>>>((double2*)s->amps, half, 1ULL << target, (const double2*)dm, ua, nrm);
    }
    cudaError_t e = cudaStreamSynchronize(s->stream);
    cudaFree(dm);
    if (e != cudaSuccess) {
        return cuda_fail(e, "uniformly_controlled");
    }
    s->stats.kernel_launches++;
    return B200SV_OK;
}

int b200sv_apply_m(b200sv_t s, uint64_t mask, uint64_t result, double nre, double nim)
{
    SV_ENTER(s);
    if (!s->amps) {
        return B200SV_OK;
    }
    SV_TRY(flush_queue(s));
    const uint64_t n = s->dim();
    const unsigned grid = stream_grid(s->dev, n, 256);
    DISPATCH_PREC(s, (k_apply_m<float><<<grid, 256, 0, s->stream>>>((float2*)s->amps, n, mask, result, make_float2((float)nre, (float)nim))),
        (k_apply_m<double><<<grid, 256, 0, s->stream>>>((double2*)s->amps, n, mask, result, make_double2(nre, nim))));
    SV_CUDA(cudaGetLastError());
    s->stats.kernel_launches++;
    return B200SV_OK;
}

int b200sv_collapse_parity(b200sv_t s, uint64_t mask, int result, double* kept)
{
    SV_ENTER(s);
    if (mask >= s->dim()) {
        return einval("ForceMParity mask out-of-bounds!");
    }
    if (!s->amps) {
        if (kept) {
            *kept = 0;
        }
        return B200SV_OK;
    }
    SV_TRY(flush_queue(s));
    const uint64_t n = s->dim();
    const unsigned grid = stream_grid(s->dev, n, 256);
    SV_CUDA(cudaMemsetAsync(s->d_scratch, 0, sizeof(double), s->stream));
    DISPATCH_PREC(s, (k_collapse_parity<float><<<grid, 256, 0, s->stream>>>((float2*)s->amps, n, mask, result ? 1 : 0, s->d_scratch)),
        (k_collapse_parity<double><<<grid, 256, 0, s->stream>>>((double2*)s->amps, n, mask, result ? 1 : 0, s->d_scratch)));
    SV_CUDA(cudaGetLastError());
    s->stats.kernel_launches++;
    SV_TRY(read_scratch(s, 1));
    if (kept) {
        *kept = s->h_scratch[0];
    }
    return B200SV_OK;
}

// ---- reductions --------------------------------------------------------------------------------------------------

int b200sv_prob_mask(b200sv_t s, uint64_t mask, uint64_t perm, double* out)
{
    SV_ENTER_RO(s);
    if (!out) {
        return einval("null out pointer");
    }
    if (mask >= s->dim() || (perm & ~mask)) {
        return einval("ProbMask mask out-of-bounds!");
    }
    SV_TRY(flush_queue(s));
    if (!s->amps) {
        *out = 0;
        return B200SV_OK;
    }
    const uint64_t n = s->dim();
    if (mask && !(mask & (mask - 1U)) && !s->external && s->nq >= 3 && s->nq <= 40) {
        // single-qubit probability: served from the memoised marginals (one sweep computes every qubit's; callers
        // such as QUnit or a measurement loop ask for many qubits between two state changes)
        if (!s->margValid) {
            SV_CUDA(cudaMemsetAsync(s->d_scratch, 0, 65 * sizeof(double), s->stream));
            const int cl = s->nq - (s->prec == 32 ? 1 : 0); // log2 of the number of 16-byte chunks
            if (cl >= 14) {
                // coalesced version: power-of-two grid, at least 4 and at most 2^20 chunks per thread
                int gBits = std::min(cl - 8 - 2, 11); // at least 4 chunks per thread
                const int itBits = cl - 8 - gBits;
                if (itBits > 20) {
                    gBits += itBits - 20;
                }
                const int itB = cl - 8 - gBits;
                DISPATCH_PREC(s, (k_prob_all_bits2<float, 20><<<1U << gBits, 256, 0, s->stream>>>((const float2*)s->amps, itB, gBits, s->nq, s->d_scratch)),
                    (k_prob_all_bits2<double, 20><<<1U << gBits, 256, 0, s->stream>>>((const double2*)s->amps, itB, gBits, s->nq, s->d_scratch)));
            } else {
                const unsigned grid = std::min<unsigned>(stream_grid(s->dev, n >> 3, 256), (unsigned)sm_count(s->dev) * 8U);
                DISPATCH_PREC(s, (k_prob_all_bits<float><<<grid, 256, 0, s->stream>>>((const float2*)s->amps, n, s->nq, s->d_scratch)),
                    (k_prob_all_bits<double><<<grid, 256, 0, s->stream>>>((const double2*)s->amps, n, s->nq, s->d_scratch)));
            }
            SV_CUDA(cudaGetLastError());
            s->stats.kernel_launches++;
            SV_TRY(read_scratch(s, 65));
            memcpy(s->marg, s->h_scratch, 65 * sizeof(double));
            s->margValid = true;
        }
        const int bit = __builtin_ctzll(mask);
        *out = perm ? s->marg[bit] : (s->marg[64] - s->marg[bit]);
        return B200SV_OK;
    }
    SV_CUDA(cudaMemsetAsync(s->d_scratch, 0, sizeof(double), s->stream));
    // subset iteration when every mask bit is >= 2^4 (reads stay >= 128 B contiguous); else predicate scan
    if (mask && !(mask & 15U)) {
        PowList pw;
        pw.n = 0;
        for (uint64_t m = mask; m; m &= m - 1U) {
            pw.low[pw.n++] = (m & (~m + 1U)) - 1U;
        }
        const uint64_t items = n >> pw.n;
        const unsigned grid = stream_grid(s->dev, items, 256);
        DISPATCH_PREC(s, (k_prob_mask_subset<float><<<grid, 256, 0, s->stream>>>((const float2*)s->amps, items, pw, perm, s->d_scratch)),
            (k_prob_mask_subset<double><<<grid, 256, 0, s->stream>>>((const double2*)s->amps, items, pw, perm, s->d_scratch)));
    } else {
        const unsigned grid = stream_grid(s->dev, n, 256);
        DISPATCH_PREC(s, (k_prob_mask<float><<<grid, 256, 0, s->stream>>>((const float2*)s->amps, n, mask, perm, s->d_scratch)),
            (k_prob_mask<double><<<grid, 256, 0, s->stream>>>((const double2*)s->amps, n, mask, perm, s->d_scratch)));
    }
    SV_CUDA(cudaGetLastError());
    s->stats.kernel_launches++;
    SV_TRY(read_scratch(s, 1));
    *out = s->h_scratch[0];
    return B200SV_OK;
}

int b200sv_prob_parity(b200sv_t s, uint64_t mask, double* out)
{
    SV_ENTER_RO(s);
    if (!out) {
        return einval("null out pointer");
    }
    if (mask >= s->dim()) {
        return einval("ProbParity mask out-of-bounds!");
    }
    SV_TRY(flush_queue(s));
    if (!s->amps || !mask) {
        *out = 0;
        return B200SV_OK;
    }
    const uint64_t n = s->dim();
    const unsigned grid = stream_grid(s->dev, n, 256);
    SV_CUDA(cudaMemsetAsync(s->d_scratch, 0, sizeof(double), s->stream));
    DISPATCH_PREC(s, (k_prob_parity<float><<<grid, 256, 0, s->stream>>>((const float2*)s->amps, n, mask, s->d_scratch)),
        (k_prob_parity<double><<<grid, 256, 0, s->stream>>>((const double2*)s->amps, n, mask, s->d_scratch)));
    SV_CUDA(cudaGetLastError());
    s->stats.kernel_launches++;
    SV_TRY(read_scratch(s, 1));
    *out = s->h_scratch[0];
    return B200SV_OK;
}

int b200sv_prob_mask_all(b200sv_t s, uint64_t mask, void* host_probs)
{
    SV_ENTER_RO(s);
    if (!host_probs) {
        return einval("null out pointer");
    }
    if (mask >= s->dim()) {
        return einval("ProbMaskAll mask out-of-bounds!");
    }
    const int k = __builtin_popcountll(mask);
    if (k > 28) {
        return einval("ProbMaskAll: too many mask bits");
    }
    SV_TRY(flush_queue(s));
    const size_t nb = (size_t)1 << k;
    const size_t rbytes = s->prec == 32 ? 4 : 8;
    if (!s->amps) {
        memset(host_probs, 0, nb * rbytes);
        return B200SV_OK;
    }
    double* bins = nullptr;
    SV_CUDA(cudaMalloc(&bins, nb * sizeof(double)));
    cudaMemsetAsync(bins, 0, nb * sizeof(double), s->stream);
    const uint64_t n = s->dim();
    const int useShared = nb <= 4096;
    const unsigned grid = std::min<unsigned>(stream_grid(s->dev, n, 256), (unsigned)sm_count(s->dev) * 4U);
    const size_t shm = useShared ? nb * sizeof(double) : 0;
    DISPATCH_PREC(s, (k_prob_mask_all<float><<<grid, 256, shm, s->stream>>>((const float2*)s->amps, n, mask, bins, useShared, (int)nb)),
        (k_prob_mask_all<double><<<grid, 256, shm, s->stream>>>((const double2*)s->amps, n, mask, bins, useShared, (int)nb)));
    s->stats.kernel_launches++;
    std::vector<double> hb(nb);
    cudaError_t e = cudaMemcpyAsync(hb.data(), bins, nb * sizeof(double), cudaMemcpyDeviceToHost, s->stream);
    if (e == cudaSuccess) {
        e = cudaStreamSynchronize(s->stream);
    }
    cudaFree(bins);
    if (e != cudaSuccess) {
        return cuda_fail(e, "prob_mask_all");
    }
    if (s->prec == 32) {
        for (size_t i = 0; i < nb; ++i) {
            ((float*)host_probs)[i] = (float)hb[i];
        }
    } else {
        memcpy(host_probs, hb.data(), nb * sizeof(double));
    }
    return B200SV_OK;
}

int b200sv_norm(b200sv_t s, double thresh, double* out)
{
    SV_ENTER_RO(s);
    if (!out) {
        return einval("null out pointer");
    }
    SV_TRY(flush_queue(s));
    if (!s->amps) {
        *out = 0;
        return B200SV_OK;
    }
    const uint64_t n = s->dim();
    const unsigned grid = stream_grid(s->dev, n, 256);
    SV_CUDA(cudaMemsetAsync(s->d_scratch, 0, sizeof(double), s->stream));
    DISPATCH_PREC(s, (k_norm<float><<<grid, 256, 0, s->stream>>>((const float2*)s->amps, n, (float)thresh, s->d_scratch)),
        (k_norm<double><<<grid, 256, 0, s->stream>>>((const double2*)s->amps, n, thresh, s->d_scratch)));
    SV_CUDA(cudaGetLastError());
    s->stats.kernel_launches++;
    SV_TRY(read_scratch(s, 1));
    *out = s->h_scratch[0];
    return B200SV_OK;
}

int b200sv_normalize(b200sv_t s, double nrm, double thresh, double phase_arg)
{
    SV_ENTER(s);
    if (!s->amps) {
        return B200SV_OK;
    }
    if (nrm <= 0) {
        return einval("normalize: non-positive norm");
    }
    SV_TRY(flush_queue(s));
    const uint64_t n = s->dim();
    const unsigned grid = stream_grid(s->dev, n, 256);
    if (s->prec == 32) {
        const float f = 1.0f / sqrtf((float)nrm);
        const float2 c = make_float2(f * cosf((float)phase_arg), f * sinf((float)phase_arg));
        k_normalize<float><<<grid, 256, 0, s->stream>>>((float2*)s->amps, n, c, (float)std::max(thresh, 0.0));
    } else {
        const double f = 1.0 / sqrt(nrm);
        const double2 c = make_double2(f * cos(phase_arg), f * sin(phase_arg));
        k_normalize<double><<<grid, 256, 0, s->stream>>>((double2*)s->amps, n, c, std::max(thresh, 0.0));
    }
    SV_CUDA(cudaGetLastError());
    s->stats.kernel_launches++;
    return B200SV_OK;
}

int b200sv_inner(b200sv_t a, b200sv_t b, double* re, double* im)
{
    SV_ENTER(a);
    if (!b || !re || !im) {
        return einval("null argument");
    }
    if (a->nq != b->nq || a->prec != b->prec) {
        return einval("inner: size mismatch");
    }
    {
        DevGuard g2(b->dev);
        SV_TRY(flush_queue(b));
    }
    SV_TRY(flush_queue(a));
    if (!a->amps || !b->amps) {
        *re = 0;
        *im = 0;
        return B200SV_OK;
    }
    if (a->dev != b->dev && enable_peer(a->dev, b->dev) != B200SV_OK) {
        return einval("inner: states on devices without peer access");
    }
    SV_TRY(cross_wait(a, b));
    const uint64_t n = a->dim();
    const unsigned grid = stream_grid(a->dev, n, 256);
    SV_CUDA(cudaMemsetAsync(a->d_scratch, 0, 2 * sizeof(double), a->stream));
    DISPATCH_PREC(a, (k_inner<float><<<grid, 256, 0, a->stream>>>((const float2*)a->amps, (const float2*)b->amps, n, a->d_scratch)),
        (k_inner<double><<<grid, 256, 0, a->stream>>>((const double2*)a->amps, (const double2*)b->amps, n, a->d_scratch)));
    SV_CUDA(cudaGetLastError());
    a->stats.kernel_launches++;
    SV_TRY(read_scratch(a, 2));
    *re = a->h_scratch[0];
    *im = a->h_scratch[1];
    return B200SV_OK;
}

int b200sv_expectation(b200sv_t s, int start, int length, double* out)
{
    SV_ENTER_RO(s);
    if (!out || start < 0 || length < 0 || start + length > s->nq) {
        return einval("GetExpectation range is out-of-bounds!");
    }
    SV_TRY(flush_queue(s));
    if (!s->amps) {
        *out = 0;
        return B200SV_OK;
    }
    // the sum form with perms (0, 2^p) on qubit start + p
    std::vector<int> bits(length);
    std::vector<uint64_t> perms(2 * (size_t)length);
    for (int p = 0; p < length; ++p) {
        bits[p] = start + p;
        perms[2 * p] = 0U;
        perms[2 * p + 1] = 1ULL << p;
    }
    double m[3];
    SV_TRY(launch_moments(s, false, length, bits.data(), perms.data(), nullptr, 0U, 0.0, m));
    *out = m[1];
    return B200SV_OK;
}

// argument checks shared by the two moments entries (before anything touches the state)
static int moments_args(const State* s, int k, const int* bits, const void* table, const double* out)
{
    if (k < 0 || !out || (k > 0 && (!bits || !table))) {
        return einval("moments: k < 0 or a NULL argument");
    }
    uint64_t seen = 0U;
    for (int p = 0; p < k; ++p) {
        if (bits[p] < 0 || bits[p] >= s->nq) {
            return einval("moments: qubit index out of bounds");
        }
        if ((seen >> bits[p]) & 1U) {
            return einval("moments: repeated qubit");
        }
        seen |= 1ULL << bits[p];
    }
    return B200SV_OK;
}

int b200sv_moments_bits(b200sv_t s, int k, const int* bits, const uint64_t* perms, uint64_t offset, double center, double* out)
{
    SV_ENTER_RO(s);
    SV_TRY(moments_args(s, k, bits, perms, out));
    // the largest weight must fit: offset + sum_p max(perms[2p], perms[2p + 1]) <= 2^64 - 1
    uint64_t top = offset;
    for (int p = 0; p < k; ++p) {
        const uint64_t m = std::max(perms[2 * p], perms[2 * p + 1]);
        if (m > ~top) {
            return einval("moments_bits: offset + sum of the largest perms exceeds 2^64 - 1");
        }
        top += m;
    }
    SV_TRY(flush_queue(s));
    if (!s->amps) {
        out[0] = out[1] = out[2] = 0;
        return B200SV_OK;
    }
    return launch_moments(s, false, k, bits, perms, nullptr, offset, center, out);
}

int b200sv_moments_floats(b200sv_t s, int k, const int* bits, const double* weights, double center, double* out)
{
    SV_ENTER_RO(s);
    SV_TRY(moments_args(s, k, bits, weights, out));
    SV_TRY(flush_queue(s));
    if (!s->amps) {
        out[0] = out[1] = out[2] = 0;
        return B200SV_OK;
    }
    return launch_moments(s, true, k, bits, nullptr, weights, 0U, center, out);
}

int b200sv_expectation_pauli(b200sv_t s, uint64_t x_mask, uint64_t z_mask, double* out)
{
    SV_ENTER_RO(s);
    if (!out) {
        return einval("null out pointer");
    }
    if (x_mask >= s->dim() || z_mask >= s->dim()) {
        return einval("expectation_pauli: mask out-of-bounds!");
    }
    SV_TRY(flush_queue(s));
    if (!s->amps) {
        out[0] = out[1] = 0;
        return B200SV_OK;
    }
    return launch_pauli(s, x_mask, z_mask, out);
}

int b200sv_reduced_density_matrix(b200sv_t s, int k, const int* qubits, double* out)
{
    SV_ENTER_RO(s);
    if (k < 0 || k > B200SV_RDM_MAX_QUBITS || k > s->nq || !out || (k > 0 && !qubits)) {
        return einval("reduced_density_matrix: k out of range or a NULL argument");
    }
    uint64_t seen = 0U;
    for (int p = 0; p < k; ++p) {
        if (qubits[p] < 0 || qubits[p] >= s->nq) {
            return einval("reduced_density_matrix: qubit index out of bounds");
        }
        if ((seen >> qubits[p]) & 1U) {
            return einval("reduced_density_matrix: repeated qubit");
        }
        seen |= 1ULL << qubits[p];
    }
    SV_TRY(flush_queue(s));
    const size_t words = (size_t)2 << (2 * k);
    if (!s->amps) {
        std::fill(out, out + words, 0.0);
        return B200SV_OK;
    }
    if (s->nq == 0) {
        // one amplitude, smaller than a 16-byte chunk: rho = |psi_0|^2
        double a[2] = {0.0, 0.0};
        if (s->prec == 32) {
            float f[2];
            SV_CUDA(cudaMemcpyAsync(f, s->amps, sizeof(f), cudaMemcpyDeviceToHost, s->stream));
            SV_CUDA(cudaStreamSynchronize(s->stream));
            a[0] = f[0];
            a[1] = f[1];
        } else {
            SV_CUDA(cudaMemcpyAsync(a, s->amps, sizeof(a), cudaMemcpyDeviceToHost, s->stream));
            SV_CUDA(cudaStreamSynchronize(s->stream));
        }
        out[0] = a[0] * a[0] + a[1] * a[1];
        out[1] = 0.0;
        return B200SV_OK;
    }
    return launch_rdm(s, k, qubits, out);
}

int b200sv_highest_prob(b200sv_t s, uint64_t* perm)
{
    SV_ENTER_RO(s);
    if (!perm) {
        return einval("null out pointer");
    }
    SV_TRY(flush_queue(s));
    *perm = 0;
    if (!s->amps) {
        return B200SV_OK;
    }
    const uint64_t n = s->dim();
    const unsigned grid = std::min<unsigned>(stream_grid(s->dev, n, 256), 1024U);
    SV_TRY(ensure_scratch(s, 2 * 1024));
    double* bv = s->d_scratch;
    unsigned long long* bi = (unsigned long long*)(s->d_scratch + 1024);
    DISPATCH_PREC(s, (k_argmax<float><<<grid, 256, 0, s->stream>>>((const float2*)s->amps, n, bv, bi)),
        (k_argmax<double><<<grid, 256, 0, s->stream>>>((const double2*)s->amps, n, bv, bi)));
    SV_CUDA(cudaGetLastError());
    s->stats.kernel_launches++;
    SV_TRY(read_scratch(s, 2048));
    double best = -1;
    uint64_t bidx = 0;
    for (unsigned b = 0; b < grid; ++b) {
        const double v = s->h_scratch[b];
        const uint64_t i = ((unsigned long long*)(s->h_scratch + 1024))[b];
        if (v > best || (v == best && i < bidx)) {
            best = v;
            bidx = i;
        }
    }
    *perm = bidx;
    return B200SV_OK;
}

int b200sv_sample(b200sv_t s, double rnd, uint64_t* perm)
{
    SV_ENTER(s);
    if (!perm) {
        return einval("null out pointer");
    }
    SV_TRY(flush_queue(s));
    const uint64_t n = s->dim();
    *perm = n - 1U;
    if (!s->amps) {
        return B200SV_OK;
    }
    // two-level search: per-chunk sums on the device, prefix on the host, then one chunk scanned on the host
    const uint64_t chunk = std::min<uint64_t>(n, 1ULL << 14);
    const uint64_t nchunks = n / chunk;
    SV_TRY(ensure_scratch(s, nchunks));
    const double eps = (s->prec == 32) ? 1.7763568394002505e-15 : 6.310887241768095e-30; // REAL1_EPSILON (qrack_types.hpp:206,209)
    DISPATCH_PREC(s, (k_chunk_sums<float><<<(unsigned)nchunks, 256, 0, s->stream>>>((const float2*)s->amps, chunk, (float)eps, s->d_scratch)),
        (k_chunk_sums<double><<<(unsigned)nchunks, 256, 0, s->stream>>>((const double2*)s->amps, chunk, eps, s->d_scratch)));
    SV_CUDA(cudaGetLastError());
    s->stats.kernel_launches++;
    SV_TRY(read_scratch(s, (int)nchunks));
    const double fpEps = (s->prec == 32) ? 2.98023223876953125e-08 : 5.551115123125783e-17; // FP_NORM_EPSILON
    double tot = 0;
    uint64_t lastNonzeroChunk = nchunks;
    uint64_t pick = nchunks;
    for (uint64_t c = 0; c < nchunks; ++c) {
        const double cs = s->h_scratch[c];
        if (cs > 0) {
            lastNonzeroChunk = c;
            if ((tot + cs > rnd) || ((1.0 - (tot + cs)) <= fpEps)) {
                pick = c;
                break;
            }
            tot += cs;
        }
    }
    if (pick == nchunks) {
        pick = lastNonzeroChunk;
        if (pick == nchunks) {
            return B200SV_OK; // all-zero state: last index (reference MAll falls through to lastNonzero = max)
        }
        tot -= 0; // scan that chunk for its last nonzero entry below
    }
    const size_t ab = s->amp_bytes();
    std::vector<char> host(chunk * ab);
    SV_CUDA(cudaMemcpyAsync(host.data(), (char*)s->amps + pick * chunk * ab, chunk * ab, cudaMemcpyDeviceToHost, s->stream));
    SV_CUDA(cudaStreamSynchronize(s->stream));
    uint64_t lastNz = n - 1U;
    bool found = false;
    for (uint64_t i = 0; i < chunk; ++i) {
        double p;
        if (s->prec == 32) {
            const float2 v = ((float2*)host.data())[i];
            p = (double)(v.x * v.x + v.y * v.y);
        } else {
            const double2 v = ((double2*)host.data())[i];
            p = v.x * v.x + v.y * v.y;
        }
        if (p > eps) {
            tot += p;
            lastNz = pick * chunk + i;
            if ((tot > rnd) || ((1.0 - tot) <= fpEps)) {
                *perm = lastNz;
                found = true;
                break;
            }
        }
    }
    if (!found) {
        *perm = lastNz;
    }
    return B200SV_OK;
}


// Multi-shot sampling of the whole register without collapse (SURVEY 8f N1; QEngine::MultiShotMeasureMask,
// src/qengine/qengine.cpp:542-609, draws from the 2^k histogram of the measured bits — here the k-bit outcome is read off a
// sampled basis state, which has the same distribution and needs neither the histogram nor a 2^n device->host copy).
// rnds[i] in [0, 1): shot i returns what b200sv_sample(s, rnds[i]) returns: the first index whose cumulative probability
// exceeds rnds[i] or comes within FP_NORM_EPSILON of 1 (the search of MAll, state.cpp:2026-2050).  ONE chunk-sum sweep serves
// every shot; each distinct chunk that holds a shot is copied once.
int b200sv_sample_many(b200sv_t s, int n_shots, const double* rnds, uint64_t* perms)
{
    SV_ENTER_RO(s);
    if (n_shots < 0 || (n_shots && (!rnds || !perms))) {
        return einval("sample_many: null argument");
    }
    SV_TRY(flush_queue(s));
    const uint64_t n = s->dim();
    const double fpEps = (s->prec == 32) ? 2.98023223876953125e-08 : 5.551115123125783e-17; // FP_NORM_EPSILON
    for (int i = 0; i < n_shots; ++i) {
        perms[i] = n - 1U;
    }
    if (!s->amps || !n_shots) {
        return B200SV_OK;
    }
    const uint64_t chunk = std::min<uint64_t>(n, 1ULL << 14);
    const uint64_t nchunks = n / chunk;
    SV_TRY(ensure_scratch(s, nchunks));
    const double eps = (s->prec == 32) ? 1.7763568394002505e-15 : 6.310887241768095e-30;
    DISPATCH_PREC(s, (k_chunk_sums<float><<<(unsigned)nchunks, 256, 0, s->stream>>>((const float2*)s->amps, chunk, (float)eps, s->d_scratch)),
        (k_chunk_sums<double><<<(unsigned)nchunks, 256, 0, s->stream>>>((const double2*)s->amps, chunk, eps, s->d_scratch)));
    SV_CUDA(cudaGetLastError());
    s->stats.kernel_launches++;
    SV_TRY(read_scratch(s, (int)nchunks));
    // shots in ascending order of rnd walk the chunk prefix sums once
    std::vector<int> order((size_t)n_shots);
    for (int i = 0; i < n_shots; ++i) {
        order[(size_t)i] = i;
    }
    std::sort(order.begin(), order.end(), [&](int a, int b) { return rnds[a] < rnds[b]; });
    std::vector<double> prefix(nchunks + 1, 0.0);
    uint64_t lastNonzeroChunk = nchunks;
    for (uint64_t c = 0; c < nchunks; ++c) {
        prefix[c + 1] = prefix[c] + s->h_scratch[c];
        if (s->h_scratch[c] > 0) {
            lastNonzeroChunk = c;
        }
    }
    if (lastNonzeroChunk == nchunks) {
        return B200SV_OK; // all-zero state
    }
    const size_t ab = s->amp_bytes();
    std::vector<char> host(chunk * ab);
    uint64_t loaded = nchunks, c = 0;
    for (int k = 0; k < n_shots; ++k) {
        const int i = order[(size_t)k];
        const double r = rnds[i];
        while (c < lastNonzeroChunk && !(prefix[c + 1] > r) && !((1.0 - prefix[c + 1]) <= fpEps)) {
            ++c;
        }
        if (loaded != c) {
            SV_CUDA(cudaMemcpyAsync(host.data(), (char*)s->amps + c * chunk * ab, chunk * ab, cudaMemcpyDeviceToHost, s->stream));
            SV_CUDA(cudaStreamSynchronize(s->stream));
            loaded = c;
        }
        double tot = prefix[c];
        uint64_t lastNz = c * chunk, pick = n;
        for (uint64_t j = 0; j < chunk; ++j) {
            double p;
            if (s->prec == 32) {
                const float2 v = ((float2*)host.data())[j];
                p = (double)(v.x * v.x + v.y * v.y);
            } else {
                const double2 v = ((double2*)host.data())[j];
                p = v.x * v.x + v.y * v.y;
            }
            if (p > eps) {
                tot += p;
                lastNz = c * chunk + j;
                if ((tot > r) || ((1.0 - tot) <= fpEps)) {
                    pick = lastNz;
                    break;
                }
            }
        }
        perms[i] = (pick == n) ? lastNz : pick;
    }
    return B200SV_OK;
}

// ---- structure ---------------------------------------------------------------------------------------------------------

int b200sv_compose(b200sv_t a, b200sv_t b, int start)
{
    SV_ENTER(a);
    if (!b) {
        return einval("null handle");
    }
    if (a->prec != b->prec) {
        return einval("Compose: precision mismatch");
    }
    if (start < 0 || start > a->nq) {
        return einval("Compose start index is out-of-bounds!");
    }
    if (a->external) {
        return einval("Compose on an external buffer");
    }
    {
        DevGuard g2(b->dev);
        SV_TRY(flush_queue(b));
    }
    SV_TRY(flush_queue(a));
    if (!b->nq) {
        return B200SV_OK;
    }
    const int nq = a->nq + b->nq;
    if (nq > 40) {
        return einval("Compose: too many qubits");
    }
    if (!a->amps || !b->amps) {
        free_amps(a);
        a->nq = nq;
        return B200SV_OK;
    }
    if (a->dev != b->dev && enable_peer(a->dev, b->dev) != B200SV_OK) {
        return einval("Compose: states on devices without peer access");
    }
    const uint64_t n = 1ULL << nq;
    void* out = nullptr;
    cudaError_t e = state_buf_alloc(a->dev, n * a->amp_bytes(), &out);
    if (e != cudaSuccess) {
        return cuda_fail(e, "cudaMalloc(compose)");
    }
    {
        const int rcw = cross_wait(a, b);
        if (rcw != B200SV_OK) {
            cudaFree(out);
            return rcw;
        }
    }
    const uint64_t startMask = (1ULL << start) - 1U;
    const uint64_t midMask = ((1ULL << b->nq) - 1U) << start;
    const uint64_t endMask = (n - 1U) & ~(startMask | midMask);
    const unsigned grid = stream_grid(a->dev, n, 256);
    DISPATCH_PREC(a, (k_compose<float><<<grid, 256, 0, a->stream>>>((float2*)out, (const float2*)a->amps, (const float2*)b->amps, n, startMask, midMask, endMask, start, b->nq)),
        (k_compose<double><<<grid, 256, 0, a->stream>>>((double2*)out, (const double2*)a->amps, (const double2*)b->amps, n, startMask, midMask, endMask, start, b->nq)));
    e = cudaGetLastError();
    a->stats.kernel_launches++;
    if (e != cudaSuccess) {
        cudaFree(out);
        return cuda_fail(e, "compose kernel");
    }
    SV_TRY(cross_wait(b, a));
    free_amps(a); // synchronises a's stream first
    a->amps = out;
    a->amps_bytes = n * a->amp_bytes();
    a->nq = nq;
    return B200SV_OK;
}

int b200sv_dispose_perm(b200sv_t s, int start, int length, uint64_t perm)
{
    SV_ENTER(s);
    if (start < 0 || length < 0 || start + length > s->nq) {
        return einval("Dispose range is out-of-bounds!");
    }
    if (!length) {
        return B200SV_OK;
    }
    if (s->external) {
        return einval("Dispose on an external buffer");
    }
    SV_TRY(flush_queue(s));
    const int nl = s->nq - length;
    if (!s->amps) {
        s->nq = nl;
        return B200SV_OK;
    }
    const uint64_t rem = 1ULL << nl;
    void* out = nullptr;
    cudaError_t e = state_buf_alloc(s->dev, rem * s->amp_bytes(), &out);
    if (e != cudaSuccess) {
        return cuda_fail(e, "cudaMalloc(dispose)");
    }
    const unsigned grid = stream_grid(s->dev, rem, 256);
    const uint64_t skipMask = (1ULL << start) - 1U;
    DISPATCH_PREC(s, (k_dispose_perm<float><<<grid, 256, 0, s->stream>>>((float2*)out, (const float2*)s->amps, rem, skipMask, length, perm << start)),
        (k_dispose_perm<double><<<grid, 256, 0, s->stream>>>((double2*)out, (const double2*)s->amps, rem, skipMask, length, perm << start)));
    e = cudaGetLastError();
    s->stats.kernel_launches++;
    if (e != cudaSuccess) {
        cudaFree(out);
        return cuda_fail(e, "dispose kernel");
    }
    free_amps(s);
    s->amps = out;
    s->amps_bytes = rem * s->amp_bytes();
    s->nq = nl; // (the reference sets qubitCount 1 when nl==0, state.cpp:1741-1745; the adapter handles that)
    return B200SV_OK;
}

int b200sv_decompose(b200sv_t s, int start, int length, b200sv_t dest)
{
    SV_ENTER(s);
    if (dest) {
        dest->margValid = false;
    }
    if (start < 0 || length < 0 || start + length > s->nq) {
        return einval("DecomposeDispose range is out-of-bounds!");
    }
    if (!length) {
        return B200SV_OK;
    }
    if (s->external || (dest && dest->external)) {
        return einval("Decompose on an external buffer");
    }
    if (dest && (dest->prec != s->prec || dest->nq != length)) {
        return einval("Decompose: destination size/precision mismatch");
    }
    SV_TRY(flush_queue(s));
    if (dest) {
        DevGuard g2(dest->dev);
        dest->queue.clear();
    }
    const int nl = s->nq - length;
    if (!s->amps) {
        s->nq = nl;
        if (dest) {
            SV_TRY(b200sv_zero(dest));
        }
        return B200SV_OK;
    }
    if (!nl) {
        // hand the buffer over (reference state.cpp:1572-1579)
        if (dest) {
            if (dest->dev != s->dev) {
                SV_TRY(b200sv_copy_page(dest, s, 0, 0, s->dim()));
                free_amps(s);
            } else {
                SV_CUDA(cudaStreamSynchronize(s->stream));
                free_amps(dest);
                dest->amps = s->amps;
                dest->amps_bytes = s->amps_bytes;
                s->amps = nullptr;
                s->amps_bytes = 0;
            }
        } else {
            free_amps(s);
        }
        s->nq = 0;
        return B200SV_OK;
    }
    const uint64_t n = s->dim();
    const uint64_t partPower = 1ULL << length, remPower = 1ULL << nl;
    const double floorv = (s->prec == 32) ? 1.7763568394002505e-15 : 6.310887241768095e-30; // amplitudeFloor = REAL1_EPSILON (qrack_types.hpp:206,209)
    const size_t ab = s->amp_bytes();
    const bool onePass = (partPower <= 2048 || remPower <= 2048);
    const bool smallIsPart = partPower <= remPower;
    void* nout = nullptr; // the remainder state
    void* pout = nullptr; // the part state (only if dest)
    double* acc = nullptr;
    cudaError_t e = state_buf_alloc(s->dev, remPower * ab, &nout);
    if (e != cudaSuccess) {
        return cuda_fail(e, "cudaMalloc(decompose remainder)");
    }
    if (dest) {
        e = state_buf_alloc(s->dev, partPower * ab, &pout);
        if (e != cudaSuccess) {
            state_buf_free(s->dev, nout, remPower * ab);
            return cuda_fail(e, "cudaMalloc(decompose part)");
        }
    }
    auto fail = [&](cudaError_t err, const char* what) {
        cudaStreamSynchronize(s->stream);
        if (acc) {
            cudaFree(acc);
        }
        state_buf_free(s->dev, nout, remPower * ab);
        if (pout) {
            state_buf_free(s->dev, pout, partPower * ab);
        }
        return cuda_fail(err, what);
    };
    if (onePass) {
        // one read of the state: the large side is rebuilt in the kernel, the small side from its bins afterwards
        const uint64_t smallN = smallIsPart ? partPower : remPower, largeN = smallIsPart ? remPower : partPower;
        const bool needSmall = smallIsPart ? (dest != nullptr) : true;
        const bool needLarge = smallIsPart ? true : (dest != nullptr);
        void* outLarge = smallIsPart ? nout : pout;
        void* scratchLarge = nullptr;
        if (!needLarge) {
            // Dispose of a LARGE part: nothing of it is kept, but the kernel writes its rows; give it a throw-away buffer
            e = state_buf_alloc(s->dev, largeN * ab, &scratchLarge);
            if (e != cudaSuccess) {
                return fail(e, "cudaMalloc(decompose scratch)");
            }
            outLarge = scratchLarge;
        }
        e = cudaMalloc(&acc, 2 * smallN * sizeof(double));
        if (e != cudaSuccess) {
            if (scratchLarge) {
                state_buf_free(s->dev, scratchLarge, largeN * ab);
            }
            return fail(e, "cudaMalloc(decompose bins)");
        }
        cudaMemsetAsync(acc, 0, 2 * smallN * sizeof(double), s->stream);
        const unsigned grid = (unsigned)std::min<uint64_t>((largeN + 255U) / 256U, (uint64_t)sm_count(s->dev) * 8U);
        const size_t shm = needSmall ? 2 * smallN * sizeof(double) : 0;
        if (s->prec == 32) {
            if (shm > 48 * 1024) {
                cudaFuncSetAttribute(k_decompose_onepass<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
            }
            k_decompose_onepass<float><<<grid, 256, shm, s->stream>>>((const float2*)s->amps, start, length, s->nq, smallIsPart ? 1 : 0, (float)floorv,
                (float2*)outLarge, acc, acc + smallN, needSmall ? 1 : 0);
        } else {
            if (shm > 48 * 1024) {
                cudaFuncSetAttribute(k_decompose_onepass<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
            }
            k_decompose_onepass<double><<<grid, 256, shm, s->stream>>>((const double2*)s->amps, start, length, s->nq, smallIsPart ? 1 : 0, floorv,
                (double2*)outLarge, acc, acc + smallN, needSmall ? 1 : 0);
        }
        s->stats.kernel_launches++;
        void* outSmall = smallIsPart ? pout : nout;
        if (outSmall) {
            const unsigned g2 = stream_grid(s->dev, smallN, 256);
            DISPATCH_PREC(s, (k_polar_rebuild<float><<<g2, 256, 0, s->stream>>>((float2*)outSmall, smallN, acc, acc + smallN, (float)floorv)),
                (k_polar_rebuild<double><<<g2, 256, 0, s->stream>>>((double2*)outSmall, smallN, acc, acc + smallN, floorv)));
            s->stats.kernel_launches++;
        }
        e = cudaStreamSynchronize(s->stream);
        if (scratchLarge) {
            state_buf_free(s->dev, scratchLarge, largeN * ab);
        }
        if (e != cudaSuccess) {
            return fail(e, "decompose");
        }
    } else {
        // both sides large: global accumulators (double atomics), then two rebuild sweeps
        const size_t accN = 2 * remPower + 2 * partPower;
        e = cudaMalloc(&acc, accN * sizeof(double));
        if (e != cudaSuccess) {
            return fail(e, "cudaMalloc(decompose marginals)");
        }
        cudaMemsetAsync(acc, 0, accN * sizeof(double), s->stream);
        double* remProb = acc;
        double* remAngle = acc + remPower;
        double* partProb = dest ? acc + 2 * remPower : nullptr;
        double* partAngle = dest ? acc + 2 * remPower + partPower : nullptr;
        const unsigned grid = std::min<unsigned>(stream_grid(s->dev, n, 256), (unsigned)sm_count(s->dev) * 8U);
        DISPATCH_PREC(s, (k_decompose_marginals<float><<<grid, 256, 0, s->stream>>>((const float2*)s->amps, n, start, length, (float)floorv, remProb, remAngle, partProb, partAngle, 0)),
            (k_decompose_marginals<double><<<grid, 256, 0, s->stream>>>((const double2*)s->amps, n, start, length, floorv, remProb, remAngle, partProb, partAngle, 0)));
        s->stats.kernel_launches++;
        {
            const unsigned g2 = stream_grid(s->dev, remPower, 256);
            DISPATCH_PREC(s, (k_polar_rebuild<float><<<g2, 256, 0, s->stream>>>((float2*)nout, remPower, remProb, remAngle, (float)floorv)),
                (k_polar_rebuild<double><<<g2, 256, 0, s->stream>>>((double2*)nout, remPower, remProb, remAngle, floorv)));
            s->stats.kernel_launches++;
        }
        if (dest) {
            const unsigned g3 = stream_grid(s->dev, partPower, 256);
            DISPATCH_PREC(s, (k_polar_rebuild<float><<<g3, 256, 0, s->stream>>>((float2*)pout, partPower, partProb, partAngle, (float)floorv)),
                (k_polar_rebuild<double><<<g3, 256, 0, s->stream>>>((double2*)pout, partPower, partProb, partAngle, floorv)));
            s->stats.kernel_launches++;
        }
        e = cudaStreamSynchronize(s->stream);
        if (e != cudaSuccess) {
            return fail(e, "decompose");
        }
    }
    cudaFree(acc);
    acc = nullptr;
    int rc = B200SV_OK;
    if (dest) {
        // the part state was built on s's device: adopt it, or move it if dest lives elsewhere
        if (dest->dev == s->dev) {
            free_amps(dest);
            dest->amps = pout;
            dest->amps_bytes = partPower * ab;
        } else {
            DevGuard g4(dest->dev);
            rc = alloc_amps(dest, false);
            if (rc == B200SV_OK) {
                e = cudaMemcpyPeer(dest->amps, dest->dev, pout, s->dev, partPower * ab);
                if (e != cudaSuccess) {
                    rc = cuda_fail(e, "decompose peer copy");
                }
            }
            state_buf_free(s->dev, pout, partPower * ab);
        }
        pout = nullptr;
    }
    if (rc != B200SV_OK) {
        state_buf_free(s->dev, nout, remPower * ab);
        return rc;
    }
    free_amps(s);
    s->amps = nout;
    s->amps_bytes = remPower * ab;
    s->nq = nl;
    return B200SV_OK;
}

// ---- stats / timing ---------------------------------------------------------------------------------------------------

int b200sv_get_stats(b200sv_t s, b200sv_stats* out)
{
    if (!s || !out) {
        return einval("null argument");
    }
    *out = s->stats;
    return B200SV_OK;
}
int b200sv_reset_stats(b200sv_t s)
{
    if (!s) {
        return einval("null argument");
    }
    memset(&s->stats, 0, sizeof(s->stats));
    return B200SV_OK;
}

int b200sv_timer_begin(b200sv_t s)
{
    SV_ENTER_RO(s);
    SV_TRY(flush_queue(s));
    SV_CUDA(cudaEventRecord(s->ev0, s->stream));
    return B200SV_OK;
}
int b200sv_timer_end(b200sv_t s, double* ms)
{
    SV_ENTER_RO(s);
    if (!ms) {
        return einval("null out pointer");
    }
    SV_TRY(flush_queue(s));
    SV_CUDA(cudaEventRecord(s->ev1, s->stream));
    SV_CUDA(cudaEventSynchronize(s->ev1));
    float f = 0;
    SV_CUDA(cudaEventElapsedTime(&f, s->ev0, s->ev1));
    *ms = f;
    return B200SV_OK;
}

int b200sv_plan_gates(int n_qubits, int precision, int n_gates, const uint64_t* off1, const uint64_t* off2, const uint64_t* pmasks,
    const double* mats8, int* n_sweeps, int* n_passes, int* n_ops)
{
    if (n_gates < 0 || (n_gates && (!off1 || !off2 || !pmasks || !mats8)) || (precision != 32 && precision != 64) || n_qubits < 5 ||
        n_qubits > 62 || !n_sweeps || !n_passes || !n_ops) {
        return einval("plan_gates: bad arguments");
    }
    std::vector<GateOp> q((size_t)n_gates);
    for (int i = 0; i < n_gates; ++i) {
        const uint64_t diff = off1[i] ^ off2[i];
        if (!diff || (diff & (diff - 1U)) || (n_qubits < 64 && (pmasks[i] >> n_qubits)) || ((off1[i] | off2[i]) & ~pmasks[i])) {
            return einval("plan_gates: not a single-target gate");
        }
        make_gate_op(precision, off1[i], off2[i], pmasks[i], mats8 + 8 * (size_t)i, 1.0, q[(size_t)i]);
    }
    return fused_plan_gates(n_qubits, precision, q, n_sweeps, n_passes, n_ops);
}

int b200sv_emulate_fused(int n_qubits, int precision, int n_gates, const uint64_t* off1, const uint64_t* off2, const uint64_t* pmasks,
    const double* mats8, void* host_state)
{
    if (n_gates < 0 || (n_gates && (!off1 || !off2 || !pmasks || !mats8)) || !host_state || (precision != 32 && precision != 64) ||
        n_qubits < 5 || n_qubits > 30) {
        return einval("emulate_fused: bad arguments");
    }
    std::vector<GateOp> q((size_t)n_gates);
    const uint64_t dim = 1ULL << n_qubits;
    for (int i = 0; i < n_gates; ++i) {
        const uint64_t diff = off1[i] ^ off2[i];
        if (!diff || (diff & (diff - 1U)) || pmasks[i] >= dim || ((off1[i] | off2[i]) & ~pmasks[i])) {
            return einval("emulate_fused: not a single-target gate");
        }
        make_gate_op(precision, off1[i], off2[i], pmasks[i], mats8 + 8 * (size_t)i, 1.0, q[(size_t)i]);
    }
    return fused_emulate(n_qubits, precision, q, host_state);
}

int b200sv_emulate_fused_pull(int n_qubits, int precision, int n_gates, const uint64_t* off1, const uint64_t* off2,
    const uint64_t* pmasks, const double* mats8, int k, const int* victim_bits, int rank, void* const* src_states, void* out_state)
{
    if (n_gates < 0 || (n_gates && (!off1 || !off2 || !pmasks || !mats8)) || (precision != 32 && precision != 64) || n_qubits < 5 ||
        n_qubits > 30) {
        return einval("emulate_fused_pull: bad arguments");
    }
    PullArgs pa;
    SV_TRY(fill_pull_args(n_qubits, precision, k, victim_bits, rank, src_states, out_state, &pa));
    std::vector<GateOp> q((size_t)n_gates);
    const uint64_t dim = 1ULL << n_qubits;
    for (int i = 0; i < n_gates; ++i) {
        const uint64_t diff = off1[i] ^ off2[i];
        if (!diff || (diff & (diff - 1U)) || pmasks[i] >= dim || ((off1[i] | off2[i]) & ~pmasks[i])) {
            return einval("emulate_fused_pull: not a single-target gate");
        }
        make_gate_op(precision, off1[i], off2[i], pmasks[i], mats8 + 8 * (size_t)i, 1.0, q[(size_t)i]);
    }
    return fused_emulate(n_qubits, precision, q, out_state, &pa);
}

int b200sv_flush_l2(b200sv_t s, uint64_t bytes)
{
    SV_ENTER_RO(s);
    bytes = (bytes + 15U) & ~15ULL;
    if (s->flush_bytes < bytes) {
        if (s->d_flush) {
            cudaFree(s->d_flush);
            s->d_flush = nullptr;
            s->flush_bytes = 0;
        }
        SV_CUDA(cudaMalloc(&s->d_flush, bytes));
        s->flush_bytes = bytes;
    }
    const uint64_t n16 = bytes / 16;
    k_fill_bytes<<<stream_grid(s->dev, n16, 256), 256, 0, s->stream>>>((uint4*)s->d_flush, n16, 0x5a5a5a5aU);
    SV_CUDA(cudaGetLastError());
    return B200SV_OK;
}

#include "alu_abi.inl"

} // extern "C"
