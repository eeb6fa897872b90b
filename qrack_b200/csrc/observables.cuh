// observables.cuh — the QInterface observable queries (reference src/qinterface/qinterface.cpp:478-800) as read-only sweeps.
//
// The reference answers ExpectationBitsFactorized / ExpectationFloatsFactorized (and, through them, ExpectationBitsAll, the
// Variance forms, ExpVarUnitaryAll and ExpectationPauliAll) with a host loop over all 2^n basis states that asks ProbAll(i) for
// each — one device round trip per basis state on a GPU engine.  Here each query is one pass over the amplitudes:
//   * k_moments: the weighted moments (S0, S1, S2) = sum_i |psi_i|^2 (1, w_i - c, (w_i - c)^2) of a weight w_i that depends
//     on the bits of i at k listed qubits, either as a sum (w_i = offset + sum_p perms[2p + bit(i, bits[p])], uint64, exact) or
//     as a product (w_i = prod_p weights[2p + bit(i, bits[p])]).  The per-qubit terms are folded into one 256-entry table per
//     index byte that holds a listed qubit (at most 8), so w_i costs one shared-memory lookup per such byte whatever k is.
//   * k_pauli: <psi|P|psi> of a Pauli string P given as (x, z) masks (X on x & ~z, Y on x & z, Z on z & ~x) without the basis
//     gates the reference applies and undoes around the Floats query: P|j> = i^|y| (-1)^popcount(j & z) |j ^ x>, so every
//     pair (j, j ^ x) is visited once (the pairing of k_xmask) and contributes twice the real part of its term.
//   * k_pauli_pair: the same term when the two members of a pair live in different buffers (a sharded state whose Pauli
//     string has X or Y on a rank-bit qubit pairs this rank's page with a partner page), read-only on both.
// All of them read each 16-byte chunk once, accumulate every term in double, and issue one atomic per CTA and output.
// Included by b200sv.cu (same translation unit as the other kernels).
#pragma once

#include <vector>

namespace b200sv {

// byte positions of the tables a moments sweep uses (table t serves index bits shift[t] .. shift[t] + 7)
struct MomTabs {
    int n;
    int shift[8];
};

template <typename R, bool PROD>
__global__ void __launch_bounds__(256) k_moments(const typename Cx<R>::type* __restrict__ psi, uint64_t n,
    const void* __restrict__ tabsGlobal, MomTabs mt, uint64_t baseSum, double center, double* out)
{
    typedef typename Cx<R>::type C;
    typedef typename std::conditional<PROD, double, uint64_t>::type W;
    extern __shared__ __align__(16) unsigned char momSmem[];
    W* tab = reinterpret_cast<W*>(momSmem);
    for (int t = threadIdx.x; t < (mt.n << 8); t += blockDim.x) {
        tab[t] = reinterpret_cast<const W*>(tabsGlobal)[t];
    }
    __syncthreads();
    double s0 = 0, s1 = 0, s2 = 0;
    auto add = [&](W w, double p) {
        const double d = (double)w - center;
        const double pd = p * d;
        s0 += p;
        s1 += pd;
        s2 += pd * d;
    };
    auto fold = [](W& w, W e) {
        if (PROD) {
            w *= e;
        } else {
            w += e;
        }
    };
    if (sizeof(R) == 4 && n >= 2) {
        // fp32: the two amplitudes of a 16-byte chunk differ in bit 0 only, so every table but the one of byte 0 is looked up
        // once per chunk, and that one's two neighbouring entries come in one 16-byte load
        typedef typename std::conditional<PROD, double2, ulonglong2>::type W2;
        const float4* p4 = reinterpret_cast<const float4*>(psi);
        const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
        for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < (n >> 1); j += stride) {
            const float4 v = p4[j];
            const uint64_t i = 2U * j;
            W wa = PROD ? (W)1 : (W)baseSum, wb = wa;
            for (int t = 0; t < mt.n; ++t) {
                const int e = (t << 8) | (int)((i >> mt.shift[t]) & 255U);
                if (mt.shift[t] == 0) {
                    const W2 pr = *reinterpret_cast<const W2*>(tab + e);
                    fold(wa, (W)pr.x);
                    fold(wb, (W)pr.y);
                } else {
                    const W x = tab[e];
                    fold(wa, x);
                    fold(wb, x);
                }
            }
            add(wa, (double)v.x * (double)v.x + (double)v.y * (double)v.y);
            add(wb, (double)v.z * (double)v.z + (double)v.w * (double)v.w);
        }
    } else {
        for_amps<R>(psi, n, [&](uint64_t i, C a) {
            W w = PROD ? (W)1 : (W)baseSum;
            for (int t = 0; t < mt.n; ++t) {
                fold(w, tab[(t << 8) | (int)((i >> mt.shift[t]) & 255U)]);
            }
            add(w, (double)a.x * (double)a.x + (double)a.y * (double)a.y);
        });
    }
    block_atomic_add(s0, out);
    block_atomic_add(s1, out + 1);
    block_atomic_add(s2, out + 2);
}

// conj(b) * a, signed, into (re, im); the i^|y| factor is applied on the host
template <typename C>
__device__ __forceinline__ void pauli_term(const C a, const C b, bool neg, double& re, double& im)
{
    const double tr = (double)b.x * (double)a.x + (double)b.y * (double)a.y;
    const double ti = (double)b.x * (double)a.y - (double)b.y * (double)a.x;
    re += neg ? -tr : tr;
    im += neg ? -ti : ti;
}
template <typename C> __device__ __forceinline__ double norm_d(const C a) { return (double)a.x * (double)a.x + (double)a.y * (double)a.y; }

// out[0] = sum |psi|^2, out[1] / out[2] = sum over pairs (j, j ^ x) with the top bit of x clear in j of
// (-1)^popcount(j & z) * Re / Im (conj(psi[j ^ x]) psi[j]); for x == 0, out[1] = sum (-1)^popcount(j & z) |psi_j|^2.
// fp32 works on 16-byte chunks (amplitudes 2c, 2c + 1): x == 1 pairs the two halves of a chunk, any other x pairs chunk c with
// chunk c ^ (x >> 1); fp64 pairs amplitudes.  `items` = chunks (x == 0, fp32 x == 1) or chunk pairs; `topLow` = 2^top - 1 for
// the top bit of the chunk-level mask.
template <typename R>
__global__ void __launch_bounds__(256) k_pauli(const typename Cx<R>::type* __restrict__ psi, uint64_t n, uint64_t items,
    uint64_t x, uint64_t z, uint64_t topLow, double* out)
{
    typedef typename Cx<R>::type C;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint64_t gid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    double s0 = 0, re = 0, im = 0;
    if (!x) {
        for_amps<R>(psi, n, [&](uint64_t i, C a) {
            const double p = norm_d(a);
            s0 += p;
            re += (__popcll(i & z) & 1) ? -p : p;
        });
    } else if (sizeof(R) == 4 && n >= 2) {
        const float4* p = reinterpret_cast<const float4*>(psi);
        const uint64_t xc = x >> 1;
        for (uint64_t j = gid; j < items; j += stride) {
            float2 a[2], b[2];
            uint64_t c;
            if (!xc) {
                c = j;
                const float4 v = p[c];
                a[0] = make_float2(v.x, v.y);
                b[0] = make_float2(v.z, v.w);
                s0 += norm_d(a[0]) + norm_d(b[0]);
                pauli_term(a[0], b[0], __popcll((2U * c) & z) & 1, re, im);
                continue;
            }
            const uint64_t lo = j & topLow;
            c = ((j ^ lo) << 1) | lo; // top bit of xc clear
            const float4 u = p[c], v = p[c ^ xc];
            a[0] = make_float2(u.x, u.y);
            a[1] = make_float2(u.z, u.w);
            b[0] = make_float2(v.x, v.y);
            b[1] = make_float2(v.z, v.w);
            s0 += norm_d(a[0]) + norm_d(a[1]) + norm_d(b[0]) + norm_d(b[1]);
            const int f = (int)(x & 1U);
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                pauli_term(a[e], b[e ^ f], __popcll((2U * c + e) & z) & 1, re, im);
            }
        }
    } else {
        for (uint64_t j = gid; j < items; j += stride) {
            const uint64_t lo = j & topLow;
            const uint64_t i = ((j ^ lo) << 1) | lo; // top bit of x clear
            const C a = psi[i], b = psi[i ^ x];
            s0 += norm_d(a) + norm_d(b);
            pauli_term(a, b, __popcll(i & z) & 1, re, im);
        }
    }
    block_atomic_add(s0, out);
    block_atomic_add(re, out + 1);
    block_atomic_add(im, out + 2);
}

// Cross-page Pauli term: out[0] / out[1] = Re / Im sum_j (-1)^popcount(j & z) conj(phi[j ^ x]) psi[j], out[2] = sum |psi|^2.
// The pair (j, j ^ x) has one member in each buffer, so unlike k_pauli every j is visited and both buffers are read once.
// fp32 works on 16-byte chunks: chunk c of psi meets chunk c ^ (x >> 1) of phi, whose two amplitudes swap when bit 0 of x is
// set; fp64 (and a one-amplitude fp32 state) pairs amplitudes.
template <typename R>
__global__ void __launch_bounds__(256) k_pauli_pair(const typename Cx<R>::type* __restrict__ psi,
    const typename Cx<R>::type* __restrict__ phi, uint64_t n, uint64_t x, uint64_t z, double* out)
{
    typedef typename Cx<R>::type C;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint64_t gid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    double s0 = 0, re = 0, im = 0;
    if (sizeof(R) == 4 && n >= 2) {
        const float4* p = reinterpret_cast<const float4*>(psi);
        const float4* q = reinterpret_cast<const float4*>(phi);
        const uint64_t xc = x >> 1;
        const int f = (int)(x & 1U);
        for (uint64_t c = gid; c < (n >> 1); c += stride) {
            const float4 u = p[c], v = q[c ^ xc];
            const float2 a[2] = {make_float2(u.x, u.y), make_float2(u.z, u.w)};
            const float2 b[2] = {make_float2(v.x, v.y), make_float2(v.z, v.w)};
            s0 += norm_d(a[0]) + norm_d(a[1]);
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                pauli_term(a[e], b[e ^ f], __popcll((2U * c + e) & z) & 1, re, im);
            }
        }
    } else {
        for (uint64_t i = gid; i < n; i += stride) {
            const C a = psi[i], b = phi[i ^ x];
            s0 += norm_d(a);
            pauli_term(a, b, __popcll(i & z) & 1, re, im);
        }
    }
    block_atomic_add(re, out);
    block_atomic_add(im, out + 1);
    block_atomic_add(s0, out + 2);
}

// One moments sweep (arguments already validated; the state is non-zero and flushed).  out[0..2] = S0, S1, S2.
static int launch_moments(State* s, bool prod, int k, const int* bits, const uint64_t* perms, const double* weights,
    uint64_t offset, double center, double* out)
{
    MomTabs mt{};
    int tabOf[8];
    for (int b = 0; b < 8; ++b) {
        tabOf[b] = -1;
    }
    for (int p = 0; p < k; ++p) {
        const int byte = bits[p] >> 3;
        if (tabOf[byte] < 0) {
            tabOf[byte] = mt.n;
            mt.shift[mt.n++] = byte << 3;
        }
    }
    // words 0..3: the zeroed outputs; then mt.n tables of 256 entries (uint64 sums or double products)
    std::vector<uint64_t> up(4 + ((size_t)mt.n << 8), 0U);
    uint64_t* tu = up.data() + 4;
    double* td = reinterpret_cast<double*>(tu);
    if (prod) {
        for (size_t e = 0; e < ((size_t)mt.n << 8); ++e) {
            td[e] = 1.0;
        }
    }
    for (int p = 0; p < k; ++p) {
        const int t = tabOf[bits[p] >> 3], sh = bits[p] & 7;
        for (int e = 0; e < 256; ++e) {
            const int bit = (e >> sh) & 1;
            if (prod) {
                td[(t << 8) | e] *= weights[2 * p + bit];
            } else {
                tu[(t << 8) | e] += perms[2 * p + bit];
            }
        }
    }
    SV_TRY(ensure_scratch(s, up.size()));
    SV_CUDA(cudaMemcpyAsync(s->d_scratch, up.data(), up.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, s->stream));
    const uint64_t n = s->dim();
    const unsigned grid = stream_grid(s->dev, (s->prec == 32 && n >= 2) ? (n >> 1) : n, 256);
    const size_t shm = ((size_t)mt.n << 8) * 8U;
    const void* tabs = s->d_scratch + 4;
    SV_TRY(with_prec(s, [&](auto r) {
        using R = decltype(r);
        const typename Cx<R>::type* psi = (const typename Cx<R>::type*)s->amps;
        if (prod) {
            k_moments<R, true><<<grid, 256, shm, s->stream>>>(psi, n, tabs, mt, offset, center, s->d_scratch);
        } else {
            k_moments<R, false><<<grid, 256, shm, s->stream>>>(psi, n, tabs, mt, offset, center, s->d_scratch);
        }
        return launched(s);
    }));
    SV_TRY(read_scratch(s, 3));
    memcpy(out, s->h_scratch, 3 * sizeof(double));
    return B200SV_OK;
}

// One Pauli-string sweep (masks validated; non-zero, flushed state).  out[0] = S0, out[1] = <psi|P|psi>.
static int launch_pauli(State* s, uint64_t x, uint64_t z, double* out)
{
    const uint64_t n = s->dim();
    const bool chunks = s->prec == 32 && n >= 2;
    const uint64_t units = chunks ? (n >> 1) : n; // 16-byte chunks (fp32) or amplitudes
    const uint64_t xu = chunks ? (x >> 1) : x;    // the part of x that moves between units
    uint64_t items = units, topLow = 0;
    if (x && xu) {
        items = units >> 1;
        topLow = (1ULL << (63 - __builtin_clzll(xu))) - 1U;
    }
    const unsigned grid = stream_grid(s->dev, items, 256);
    SV_TRY(with_prec(s, [&](auto r) {
        using R = decltype(r);
        return scratch_reduce(s, 3, [&] {
            k_pauli<R><<<grid, 256, 0, s->stream>>>((const typename Cx<R>::type*)s->amps, n, items, x, z, topLow, s->d_scratch);
        });
    }));
    const double re = s->h_scratch[1], im = s->h_scratch[2];
    out[0] = s->h_scratch[0];
    if (!x) {
        out[1] = re;
        return B200SV_OK;
    }
    // Re(i^|y| * term), summed over both members of each pair
    switch (__builtin_popcountll(x & z) & 3) {
    case 0:
        out[1] = 2.0 * re;
        break;
    case 1:
        out[1] = -2.0 * im;
        break;
    case 2:
        out[1] = -2.0 * re;
        break;
    default:
        out[1] = 2.0 * im;
        break;
    }
    return B200SV_OK;
}

// One cross-page Pauli sweep (masks validated; non-zero, flushed state; partner not NULL).  out as b200sv_expectation_pauli_pair.
static int launch_pauli_pair(State* s, const void* partner, uint64_t x, uint64_t z, double* out)
{
    const uint64_t n = s->dim();
    const unsigned grid = stream_grid(s->dev, (s->prec == 32 && n >= 2) ? (n >> 1) : n, 256);
    SV_TRY(with_prec(s, [&](auto r) {
        using R = decltype(r);
        typedef typename Cx<R>::type C;
        return scratch_reduce(s, 3, [&] {
            k_pauli_pair<R><<<grid, 256, 0, s->stream>>>((const C*)s->amps, (const C*)partner, n, x, z, s->d_scratch);
        });
    }));
    memcpy(out, s->h_scratch, 3 * sizeof(double));
    return B200SV_OK;
}

} // namespace b200sv
