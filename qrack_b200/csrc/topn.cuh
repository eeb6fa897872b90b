// topn.cuh — the n most probable basis states (QInterface::HighestProbAll(n), reference src/qinterface/qinterface.cpp:962-1003)
// as a radix select over the state.
//
// The key of index i is P(i) = min(|psi_i|^2, 1), computed in double (fp32: the squares of the float components are exact
// in double, so only the sum rounds; fp64: __dadd_rn(__dmul_rn(re, re), __dmul_rn(im, im))).  The order is P descending, then
// the index ascending.  As one composite key, larger = better: the 64 bits of P (P >= 0, so its bits order like the double),
// then the nq index bits inverted.  P = 0 is never selected.
//   1. k_topn_stats reads the state once for the count of P > 0 and the smallest and largest positive P.  The bits above the
//      first one where those two differ are common to every candidate, so the digit passes start there (a uniform
//      superposition needs no P pass at all).
//   2. k_topn_hist builds the histogram of the next 11-bit digit over the entries that match the selected prefix, in shared
//      memory with warp-aggregated increments (__match_any_sync), then one global atomic per nonzero bin and CTA.  The host
//      reads it back and picks the bin holding the n-th remaining entry, scanning from the best bin down.  After the 64 P
//      bits come the index bits: ties in P go to the smaller index.
//   3. Once the prefix class fits TOPN_CAP entries, k_topn_collect writes its (P, index) pairs to a candidate buffer, and
//      every entry strictly better than the prefix to the output, in the same read.  Later digit passes read the candidates
//      instead of the state.
//   4. When the class holds exactly the entries still to take, a last k_topn_collect moves the class (and anything better not
//      yet moved) to the output.  The host sorts the n entries.
// The index part of the key can be a tie key t(i) = key_xor ^ (OR over the bits b set in i of 2^key_pos[b]), key_bits wide,
// instead of i (b200sv_highest_probs_keyed: a page of a sharded state ties by its logical index).  The keyed launches (KEY) of
// k_topn_hist / k_topn_collect stage the byte tables of the map in shared memory and look t(i) up where the prefix or an
// output entry needs it; candidates and output entries carry t(i), so the candidate passes and the host sort are unchanged.
// The identity map runs the unkeyed instantiations, today's kernels.
// Included by b200sv.cu (same translation unit as the other kernels).
#pragma once

#include <algorithm>
#include <cstring>
#include <type_traits>
#include <vector>

namespace b200sv {

static const int TOPN_THREADS = 256;
static const int TOPN_DIGIT = 11; // bits per radix digit
static const int TOPN_BINS = 1 << TOPN_DIGIT;
static const uint64_t TOPN_CAP = 1ULL << 20; // a prefix class this small is compacted into the candidate buffer
// unsigned long long words of the state's scratch: [0, TOPN_BINS) histogram; then count / min / max of P > 0 and the
// output / candidate counters; from TOPN_HEAD on the output and candidate buffers when they fit in 1 MiB.  A keyed select
// puts the key tables at TOPN_HEAD and the buffers after them, from TOPN_KEY_HEAD.
static const int TOPN_ST = TOPN_BINS, TOPN_CTR = TOPN_BINS + 3, TOPN_HEAD = TOPN_BINS + 8;
static const int TOPN_KEY_TABS = 5; // byte tables of the tie key: 40 index bits, the widest state
static const int TOPN_KEY_HEAD = TOPN_HEAD + TOPN_KEY_TABS * 256;

struct __align__(16) TopnEntry {
    unsigned long long p; // bits of P
    unsigned long long i; // basis index
};

// the selected prefix of the composite key and the next digit
struct TopnPrefix {
    uint64_t hiMask, hiVal; // resolved bits of P
    uint64_t loMask, loVal; // resolved bits of the inverted tie key, ~t << (64 - kbits)
    int word;               // the digit is in P (0) or in the inverted tie key (1)
    int shift, width;       // digit = (word >> shift) & (2^width - 1)
    int kbits;              // width of the tie key (nq for the identity)
};

// the tie key of a keyed launch: t(i) = xr ^ tab[0][i & 255] ^ tab[1][(i >> 8) & 255] ^ ..., ntab tables of 256 words
struct TopnKey {
    const unsigned long long* tab;
    unsigned long long xr;
    int ntab;
};

template <typename R> __device__ __forceinline__ uint64_t topn_pbits(R re, R im)
{
    const double x = (double)re, y = (double)im;
    return (uint64_t)__double_as_longlong(fmin(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), 1.0));
}

__device__ __forceinline__ uint64_t topn_lo(uint64_t i, int kbits) { return kbits ? (~i) << (64 - kbits) : 0U; }

// the key tables of a keyed launch, staged by topn_stage_key (dynamic shared memory of ntab * 2 KiB)
__device__ __forceinline__ unsigned long long* topn_key_smem()
{
    extern __shared__ unsigned long long topn_kt[];
    return topn_kt;
}

// every thread of the CTA copies its share of the tables; the caller syncs before the first lookup
__device__ __forceinline__ void topn_stage_key(const TopnKey& k)
{
    unsigned long long* kt = topn_key_smem();
    for (int w = threadIdx.x; w < (k.ntab << 8); w += blockDim.x) {
        kt[w] = k.tab[w];
    }
}

__device__ __forceinline__ uint64_t topn_key(uint64_t i, const TopnKey& k)
{
    const unsigned long long* kt = topn_key_smem();
    uint64_t t = k.xr;
#pragma unroll
    for (int b = 0; b < TOPN_KEY_TABS; ++b) {
        if (b < k.ntab) {
            t ^= kt[(b << 8) | (unsigned)((i >> (8 * b)) & 255U)]; // distinct positions: OR = XOR
        }
    }
    return t;
}

// the inverted index part of the key of entry i.  Keyed: t(i) is looked up only while index bits are resolved or in the
// digit (a.loMask or a.word), before that the index part does not take part in any comparison.
template <bool KEY> __device__ __forceinline__ uint64_t topn_lo_of(uint64_t i, const TopnPrefix& a, const TopnKey& k)
{
    if constexpr (KEY) {
        if (!a.loMask && a.word == 0) {
            return 0U;
        }
        i = topn_key(i, k);
    }
    return topn_lo(i, a.kbits);
}

// 1: the key is better than the prefix, 0: it is in the prefix class, -1: worse
__device__ __forceinline__ int topn_cmp(uint64_t p, uint64_t lo, const TopnPrefix& a)
{
    const uint64_t h = p & a.hiMask, l = lo & a.loMask;
    if (h != a.hiVal) {
        return h > a.hiVal ? 1 : -1;
    }
    if (l != a.loVal) {
        return l > a.loVal ? 1 : -1;
    }
    return 0;
}

// f(pbits, index) for every entry of the source, with all 32 lanes of a warp in every call (f uses full-warp intrinsics);
// lanes past the end see P = 0.  SRC 0: an fp32 state, one float4 chunk (amplitudes 2j, 2j + 1) per lane and step, as
// for_amps reads it (one float2 when the state has a single amplitude); 1: an fp64 state, one double2; 2: candidates.
template <int SRC, typename F> __device__ __forceinline__ void topn_for_entries(const void* __restrict__ src, uint64_t count, F f)
{
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint64_t lane = threadIdx.x & 31;
    const uint64_t first = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31U);
    if constexpr (SRC == 0) {
        if (count >= 2) {
            const float4* p = reinterpret_cast<const float4*>(src);
            const uint64_t m = count >> 1;
            for (uint64_t b = first; b < m; b += stride) {
                const uint64_t j = b + lane;
                const float4 v = (j < m) ? p[j] : make_float4(0.f, 0.f, 0.f, 0.f);
                f(topn_pbits<float>(v.x, v.y), 2U * j);
                f(topn_pbits<float>(v.z, v.w), 2U * j + 1U);
            }
        } else {
            const float2* p = reinterpret_cast<const float2*>(src);
            for (uint64_t b = first; b < count; b += stride) {
                const uint64_t j = b + lane;
                const float2 v = (j < count) ? p[j] : make_float2(0.f, 0.f);
                f(topn_pbits<float>(v.x, v.y), j);
            }
        }
    } else if constexpr (SRC == 1) {
        const double2* p = reinterpret_cast<const double2*>(src);
        for (uint64_t b = first; b < count; b += stride) {
            const uint64_t j = b + lane;
            const double2 v = (j < count) ? p[j] : make_double2(0.0, 0.0);
            f(topn_pbits<double>(v.x, v.y), j);
        }
    } else {
        const TopnEntry* p = reinterpret_cast<const TopnEntry*>(src);
        for (uint64_t b = first; b < count; b += stride) {
            const uint64_t j = b + lane;
            const TopnEntry e = (j < count) ? p[j] : TopnEntry{0U, 0U};
            f((uint64_t)e.p, (uint64_t)e.i);
        }
    }
}

template <typename T> __device__ __forceinline__ T topn_warp_min(T v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
    }
    return v;
}
template <typename T> __device__ __forceinline__ T topn_warp_max(T v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
    }
    return v;
}

// st[0] += count of P > 0, st[1] = min(st[1], smallest positive P), st[2] = max(st[2], largest P): one atomic each per warp
template <int SRC>
__global__ void __launch_bounds__(TOPN_THREADS) k_topn_stats(const void* __restrict__ src, uint64_t count, unsigned long long* st)
{
    unsigned long long c = 0U, mn = ~0ULL, mx = 0U;
    topn_for_entries<SRC>(src, count, [&](uint64_t p, uint64_t) {
        if (p) {
            ++c;
            mn = min(mn, (unsigned long long)p);
            mx = max(mx, (unsigned long long)p);
        }
    });
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        c += __shfl_xor_sync(0xffffffffu, c, o);
    }
    mn = topn_warp_min(mn);
    mx = topn_warp_max(mx);
    if ((threadIdx.x & 31) == 0 && c) {
        atomicAdd(st, c);
        atomicMin(st + 1, mn);
        atomicMax(st + 2, mx);
    }
}

// hist[d] += the number of entries with P > 0 in the prefix class whose next digit is d
template <int SRC, bool KEY>
__global__ void __launch_bounds__(TOPN_THREADS) k_topn_hist(const void* __restrict__ src, uint64_t count, TopnPrefix a,
    TopnKey key, unsigned long long* hist)
{
    static_assert(!KEY || SRC != 2, "candidates already carry their keys");
    __shared__ unsigned int h[TOPN_BINS];
    const unsigned bins = 1U << a.width;
    for (unsigned b = threadIdx.x; b < bins; b += TOPN_THREADS) {
        h[b] = 0U;
    }
    if constexpr (KEY) {
        topn_stage_key(key);
    }
    __syncthreads();
    const unsigned lane = threadIdx.x & 31;
    topn_for_entries<SRC>(src, count, [&](uint64_t p, uint64_t i) {
        const uint64_t lo = topn_lo_of<KEY>(i, a, key);
        const bool in = p != 0U && topn_cmp(p, lo, a) == 0;
        if (!__any_sync(0xffffffffu, in)) {
            return;
        }
        const unsigned d = (unsigned)(((a.word == 0) ? p : lo) >> a.shift) & (bins - 1U);
        // lanes with the same digit: the lowest adds for all of them
        const unsigned peers = __match_any_sync(0xffffffffu, in ? d : 0xffffffffu);
        if (in && lane == (unsigned)(__ffs(peers) - 1)) {
            atomicAdd(&h[d], (unsigned)__popc(peers));
        }
    });
    __syncthreads();
    for (unsigned b = threadIdx.x; b < bins; b += TOPN_THREADS) {
        if (h[b]) {
            atomicAdd(hist + b, (unsigned long long)h[b]);
        }
    }
}

// append (p, i) of every lane with `take` to buf at slots from *ctr on: one atomic per warp (warp-uniform control flow)
__device__ __forceinline__ void topn_push(bool take, TopnEntry* buf, unsigned long long* ctr, unsigned long long cap, uint64_t p,
    uint64_t i)
{
    const unsigned m = __ballot_sync(0xffffffffu, take);
    if (!m) {
        return;
    }
    const unsigned lane = threadIdx.x & 31, leader = __ffs(m) - 1;
    unsigned long long base = 0U;
    if (lane == leader) {
        base = atomicAdd(ctr, (unsigned long long)__popc(m));
    }
    base = __shfl_sync(0xffffffffu, base, leader);
    const unsigned long long slot = base + __popc(m & ((1U << lane) - 1U));
    // the host sized the buffers from the histograms; a count past them is reported, never written
    if (take && slot < cap) {
        buf[slot] = TopnEntry{(unsigned long long)p, (unsigned long long)i};
    }
}

// entries better than the prefix -> out; the prefix class -> cand, or to out when cand is null.  ctr[0] / ctr[1] count them.
// Both take the entry's tie key in place of its index.
template <int SRC, bool KEY>
__global__ void __launch_bounds__(TOPN_THREADS) k_topn_collect(const void* __restrict__ src, uint64_t count, TopnPrefix a,
    TopnKey key, TopnEntry* out, unsigned long long outCap, TopnEntry* cand, unsigned long long candCap, unsigned long long* ctr)
{
    static_assert(!KEY || SRC != 2, "candidates already carry their keys");
    if constexpr (KEY) {
        topn_stage_key(key);
        __syncthreads();
    }
    topn_for_entries<SRC>(src, count, [&](uint64_t p, uint64_t i) {
        const int c = p ? topn_cmp(p, topn_lo_of<KEY>(i, a, key), a) : -1;
        const bool toOut = c > 0 || (c == 0 && !cand), toCand = cand && c == 0;
        if constexpr (KEY) {
            if (__any_sync(0xffffffffu, toOut || toCand)) { // only entries that are written need their key
                i = topn_key(i, key);
            }
        }
        topn_push(toOut, out, ctr, outCap, p, i);
        if (cand) {
            topn_push(toCand, cand, ctr + 1, candCap, p, i);
        }
    });
}

template <typename K> static unsigned topn_grid(State* s, K kern, uint64_t units, size_t smem = 0)
{
    // a persistent grid: every CTA resident at once, none idle on a small source
    int perSm = 1;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, kern, TOPN_THREADS, smem);
    const uint64_t need = (units + TOPN_THREADS - 1) / TOPN_THREADS;
    return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(need, (uint64_t)sm_count(s->dev) * std::max(perSm, 1)));
}

// 16-byte units a pass over the source steps through
template <int SRC> static uint64_t topn_units(uint64_t count) { return (SRC == 0 && count >= 2) ? count >> 1 : count; }

template <int SRC> static int topn_stats(State* s, const void* src, uint64_t count)
{
    unsigned long long* st = reinterpret_cast<unsigned long long*>(s->d_scratch) + TOPN_ST;
    SV_CUDA(cudaMemsetAsync(st, 0, 3 * sizeof(unsigned long long), s->stream));
    SV_CUDA(cudaMemsetAsync(st + 1, 0xff, sizeof(unsigned long long), s->stream));
    k_topn_stats<SRC><<<topn_grid(s, k_topn_stats<SRC>, topn_units<SRC>(count)), TOPN_THREADS, 0, s->stream>>>(src, count, st);
    SV_TRY(launched(s));
    SV_CUDA(cudaMemcpyAsync(reinterpret_cast<unsigned long long*>(s->h_scratch) + TOPN_ST, st, 3 * sizeof(unsigned long long),
        cudaMemcpyDeviceToHost, s->stream));
    SV_CUDA(cudaStreamSynchronize(s->stream));
    return B200SV_OK;
}

template <bool KEY> static size_t topn_smem(const TopnKey& k) { return KEY ? (size_t)k.ntab * 256 * sizeof(unsigned long long) : 0; }

template <int SRC, bool KEY> static int topn_hist(State* s, const void* src, uint64_t count, const TopnPrefix& a, const TopnKey& k)
{
    unsigned long long* h = reinterpret_cast<unsigned long long*>(s->d_scratch);
    const size_t smem = topn_smem<KEY>(k);
    return scratch_reduce(s, 1 << a.width, [&] {
        k_topn_hist<SRC, KEY><<<topn_grid(s, k_topn_hist<SRC, KEY>, topn_units<SRC>(count), smem), TOPN_THREADS, smem, s->stream>>>(
            src, count, a, k, h);
    });
}

template <int SRC, bool KEY>
static int topn_collect(State* s, const void* src, uint64_t count, const TopnPrefix& a, const TopnKey& k, TopnEntry* out,
    uint64_t outCap, TopnEntry* cand, uint64_t candCap)
{
    unsigned long long* ctr = reinterpret_cast<unsigned long long*>(s->d_scratch) + TOPN_CTR;
    const size_t smem = topn_smem<KEY>(k);
    k_topn_collect<SRC, KEY><<<topn_grid(s, k_topn_collect<SRC, KEY>, topn_units<SRC>(count), smem), TOPN_THREADS, smem,
        s->stream>>>(src, count, a, k, out, outCap, cand, candCap, ctr);
    return launched(s);
}

// f(SRC, KEY) as std::integral_constants: the source (0 / 1: an fp32 / fp64 state, 2: candidates) and whether t(i) is looked
// up (a keyed select on the state; candidates carry their keys)
template <typename F> static int topn_dispatch(int src, bool keyed, F&& f)
{
    using S0 = std::integral_constant<int, 0>;
    using S1 = std::integral_constant<int, 1>;
    if (src == 2) {
        return f(std::integral_constant<int, 2>(), std::false_type());
    }
    if (keyed) {
        return src == 0 ? f(S0(), std::true_type()) : f(S1(), std::true_type());
    }
    return src == 0 ? f(S0(), std::false_type()) : f(S1(), std::false_type());
}

// The tie key of a select: t(i) = xr ^ (OR over the bits b set in i of 2^pos[b]), `bits` wide.  pos == nullptr means
// pos[b] = b; with that and xr == 0 the select runs the unkeyed kernels.
struct TopnMap {
    int bits;
    const int* pos;
    uint64_t xr;
};

// keys[0..n) = the tie keys of the n most probable basis states, probs[0..n) their P when probs is not null (the state is
// non-zero and flushed; 1 <= n <= 2^nq; the map was checked by the caller)
static int topn_select(State* s, uint64_t n, const TopnMap& map, uint64_t* keys, double* probs)
{
    const int state = (s->prec == 32) ? 0 : 1;
    const uint64_t dim = s->dim();
    bool keyed = map.xr != 0;
    for (int b = 0; map.pos && b < s->nq; ++b) {
        keyed = keyed || map.pos[b] != b;
    }
    const size_t head = keyed ? TOPN_KEY_HEAD : TOPN_HEAD;
    SV_TRY(ensure_scratch(s, head));
    // pass 1: the count, smallest and largest P > 0 (the index plays no part)
    SV_TRY(state == 0 ? topn_stats<0>(s, s->amps, dim) : topn_stats<1>(s, s->amps, dim));
    const unsigned long long* hs = reinterpret_cast<const unsigned long long*>(s->h_scratch);
    const uint64_t pos = hs[TOPN_ST], pmin = hs[TOPN_ST + 1], pmax = hs[TOPN_ST + 2];
    std::fill(keys, keys + n, 0U);
    if (probs) {
        std::fill(probs, probs + n, 0.0);
    }
    if (!pos) {
        return B200SV_OK;
    }
    const uint64_t outCap = std::min(n, pos);

    // the byte tables of t(i) at TOPN_HEAD of the device scratch; staged again whenever alloc grows (reallocates) the scratch
    TopnKey key{nullptr, map.xr, (s->nq + 7) / 8};
    std::vector<unsigned long long> tabs;
    size_t tabsAt = 0; // the scratch size the tables were staged into
    auto stage = [&]() -> int {
        key.tab = reinterpret_cast<const unsigned long long*>(s->d_scratch) + TOPN_HEAD;
        tabsAt = s->scratch_doubles;
        SV_CUDA(cudaMemcpyAsync(const_cast<unsigned long long*>(key.tab), tabs.data(), tabs.size() * sizeof(unsigned long long),
            cudaMemcpyHostToDevice, s->stream));
        return B200SV_OK;
    };
    if (keyed) {
        tabs.assign((size_t)key.ntab * 256, 0U);
        for (int b = 0; b < s->nq; ++b) {
            const uint64_t bit = 1ULL << (map.pos ? map.pos[b] : b);
            for (unsigned v = 0; v < 256U; ++v) {
                if ((v >> (b & 7)) & 1U) {
                    tabs[(size_t)(b >> 3) * 256 + v] |= bit;
                }
            }
        }
        SV_TRY(stage());
    }

    TopnPrefix a{};
    a.kbits = map.bits;
    int L = 0;         // resolved key bits (P: 0..63, then the index: 64..64 + nq - 1)
    uint64_t r = n;    // entries still to take from the prefix class
    uint64_t cls = pos; // entries in the prefix class
    if (pos <= n) {
        r = pos; // every P > 0 is taken: the empty prefix
    } else if (pmin == pmax) {
        L = 64; // P ties everywhere: only the index bits remain
        a.hiMask = ~0ULL;
        a.hiVal = pmax;
    } else {
        L = __builtin_clzll(pmin ^ pmax); // the bits above are the same in every P > 0
        a.hiMask = L ? (~0ULL << (64 - L)) : 0U;
        a.hiVal = pmax & a.hiMask;
    }

    int src = state;
    const void* sp = s->amps;
    uint64_t scount = dim;
    TopnEntry *dOut = nullptr, *dCand = nullptr;
    uint64_t candCap = 0U;
    DevBuf<> owned;
    // out (and the candidates) in the scratch up to 1 MiB, else in a buffer for this call only; the counters start at 0
    auto alloc = [&](uint64_t nCand) -> int {
        void* base = nullptr;
        SV_TRY(scratch_or_own(s, head, (size_t)(outCap + nCand) * sizeof(TopnEntry), owned, &base));
        if (keyed && s->scratch_doubles != tabsAt) {
            SV_TRY(stage());
        }
        dOut = static_cast<TopnEntry*>(base);
        dCand = nCand ? dOut + outCap : nullptr;
        candCap = nCand;
        SV_CUDA(cudaMemsetAsync(reinterpret_cast<unsigned long long*>(s->d_scratch) + TOPN_CTR, 0, 2 * sizeof(unsigned long long),
            s->stream));
        return B200SV_OK;
    };

    while (cls != r) {
        if (src != 2 && cls <= TOPN_CAP) {
            // the class fits: move it to the candidates, and what is better to the output, in one read of the state
            SV_TRY(alloc(cls));
            SV_TRY(topn_dispatch(src, keyed, [&](auto S, auto K) {
                return topn_collect<decltype(S)::value, decltype(K)::value>(s, sp, scount, a, key, dOut, outCap, dCand, candCap);
            }));
            src = 2;
            sp = dCand;
            scount = cls;
        }
        int w;
        if (L < 64) {
            a.word = 0;
            w = std::min(TOPN_DIGIT, 64 - L);
            a.shift = 64 - L - w;
        } else {
            a.word = 1;
            w = std::min(TOPN_DIGIT, a.kbits - (L - 64));
            a.shift = 64 - (L - 64) - w;
        }
        a.width = w;
        SV_TRY(topn_dispatch(src, keyed, [&](auto S, auto K) {
            return topn_hist<decltype(S)::value, decltype(K)::value>(s, sp, scount, a, key);
        }));
        // the bin holding the r-th remaining entry, counted from the best bin down
        const unsigned long long* cnt = reinterpret_cast<const unsigned long long*>(s->h_scratch);
        uint64_t above = 0U;
        uint64_t b = ((uint64_t)1 << w) - 1U;
        while (above + cnt[b] < r) {
            above += cnt[b];
            --b;
        }
        r -= above;
        cls = cnt[b];
        const uint64_t m = (((uint64_t)1 << w) - 1U) << a.shift;
        if (a.word == 0) {
            a.hiMask |= m;
            a.hiVal |= b << a.shift;
        } else {
            a.loMask |= m;
            a.loVal |= b << a.shift;
        }
        L += w;
    }
    // the class is exactly what is left to take: it and everything better go to the output
    if (!dOut) {
        SV_TRY(alloc(0));
    }
    SV_TRY(topn_dispatch(src, keyed, [&](auto S, auto K) {
        return topn_collect<decltype(S)::value, decltype(K)::value>(s, sp, scount, a, key, dOut, outCap, nullptr, 0);
    }));

    std::vector<TopnEntry> pageable;
    TopnEntry* h = owned ? nullptr : reinterpret_cast<TopnEntry*>(reinterpret_cast<unsigned long long*>(s->h_scratch) + TOPN_HEAD);
    if (owned) {
        pageable.resize(outCap);
        h = pageable.data();
    }
    SV_CUDA(cudaMemcpyAsync(h, dOut, outCap * sizeof(TopnEntry), cudaMemcpyDeviceToHost, s->stream));
    SV_CUDA(cudaMemcpyAsync(reinterpret_cast<unsigned long long*>(s->h_scratch) + TOPN_CTR,
        reinterpret_cast<unsigned long long*>(s->d_scratch) + TOPN_CTR, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost,
        s->stream));
    SV_CUDA(cudaStreamSynchronize(s->stream));
    hs = reinterpret_cast<const unsigned long long*>(s->h_scratch); // alloc may have grown the scratch
    if (hs[TOPN_CTR] != outCap || hs[TOPN_CTR + 1] != candCap) {
        set_error("highest_probs: the selection counted " + std::to_string(hs[TOPN_CTR]) + " entries, expected " +
            std::to_string(outCap));
        return B200SV_ESTATE;
    }
    std::sort(h, h + outCap, [](const TopnEntry& x, const TopnEntry& y) { return x.p != y.p ? x.p > y.p : x.i < y.i; });
    for (uint64_t t = 0; t < outCap; ++t) {
        keys[t] = h[t].i;
        if (probs) {
            std::memcpy(&probs[t], &h[t].p, sizeof(double));
        }
    }
    return B200SV_OK;
}

} // namespace b200sv
