// sample.cuh — MAll's search (reference state.cpp:2026-2050) for many shots at once, on the device, with the picks mapped
// through a tie key (b200sv_sample_keyed; b200sv_sample and b200sv_sample_many are the identity key).
//
// The search of shot rnd: the first index i with |psi_i|^2 > REAL1_EPSILON whose running sum tot_i (in double, from index 0
// up, adding only those terms) exceeds rnd or comes within FP_NORM_EPSILON of 1; else the last index with |psi|^2 >
// REAL1_EPSILON; else 2^n - 1.  Two levels, so that one read of the state serves every shot:
//   1. k_chunk_sums sums each 2^14-amplitude chunk; the host sorts the shots by rnd and walks the chunks' prefix once, giving
//      every shot its chunk c (the first whose prefix[c + 1] passes the test, capped at the last nonzero chunk).  The chunk
//      never decreases with rnd, so the shots of a chunk are contiguous and in ascending rnd.
//   2. k_sample_search: one CTA per chunk that holds shots.  tot starts at prefix[c] and is summed sequentially in index
//      order, so every tot_i is the double a sequential scan from prefix[c] computes.  The loader warps stage the next
//      segment of p_i (0 where p_i <= REAL1_EPSILON: adding 0 leaves tot unchanged) in shared memory while one lane walks the
//      current one.  Since tot only grows and the group is in ascending rnd, each shot's pick is at or after the previous
//      one's: one walk serves the whole group.  The walk stops when the group is served, or at the chunk's end, where the
//      rest take the chunk's last nonzero index (c * chunk if it has none).  The CTA then maps its picks through the key t(j).
// Included by b200sv.cu (same translation unit as the other kernels).
#pragma once

#include <algorithm>
#include <vector>

namespace b200sv {

static const int SAMPLE_THREADS = 128;  // warp 0 walks (one lane), warps 1..3 stage the next segment
static const int SAMPLE_SEG = 1024;     // p values per staged segment (8 KiB of doubles, two buffers)
static const int SAMPLE_BATCH = 8;      // tot values summed between two tests of the group's next shot

// t(j) = xr ^ (OR over the bits b set in j of 2^pos[b]); identity when ident
struct SampleKey {
    unsigned long long xr;
    int ident;
    unsigned char pos[64];
};

__host__ __device__ __forceinline__ uint64_t sample_key(uint64_t j, const SampleKey& k)
{
    if (k.ident) {
        return j;
    }
    uint64_t t = k.xr;
#pragma unroll
    for (int b = 0; b < 64; ++b) { // static indices: pos stays in the parameter bank (bits past the qubits are 0)
        t ^= ((j >> b) & 1U) << k.pos[b]; // distinct positions: the OR over j's bits is this XOR, and xr is XORed on top
    }
    return t;
}

// a chunk that holds shots: its index, the sum of the chunks before it, and where its shots begin in the sorted list (the
// next group's begin is where they end)
struct __align__(16) SampleGroup {
    double prefix;
    unsigned c;
    unsigned begin;
};

// p = |psi_j|^2 rounded as the host rounds it (no contraction into an FMA), 0 unless p > eps
__device__ __forceinline__ double sample_p(float2 v, double eps)
{
    const double p = (double)__fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y));
    return p > eps ? p : 0.0;
}
__device__ __forceinline__ double sample_p(double2 v, double eps)
{
    const double p = __dadd_rn(__dmul_rn(v.x, v.x), __dmul_rn(v.y, v.y));
    return p > eps ? p : 0.0;
}

// stage p of amplitudes [from, from + len) into dst, threads [t0, t0 + nt) of the CTA
template <typename C>
__device__ __forceinline__ void sample_stage(const C* __restrict__ psi, uint64_t from, int len, double eps, double* dst, int t0, int nt)
{
    for (int i = (int)threadIdx.x - t0; i < len; i += nt) {
        dst[i] = sample_p(psi[from + i], eps);
    }
}

// keys[slot[k]] = t(pick of shot k) for the shots of group blockIdx.x, whose rnds srnd[k] ascend
template <typename R>
__global__ void __launch_bounds__(SAMPLE_THREADS) k_sample_search(const typename Cx<R>::type* __restrict__ psi, uint64_t chunk,
    double eps, double fpEps, const SampleGroup* __restrict__ groups, const double* __restrict__ srnd,
    const unsigned* __restrict__ slot, unsigned long long* keys, SampleKey key)
{
    __shared__ double sp[2][SAMPLE_SEG];
    const SampleGroup g = groups[blockIdx.x];
    const unsigned end = groups[blockIdx.x + 1].begin;
    const uint64_t base = (uint64_t)g.c * chunk;
    const int seg = (chunk < (uint64_t)SAMPLE_SEG) ? (int)chunk : SAMPLE_SEG;
    const int nseg = (int)(chunk / seg);
    sample_stage(psi, base, seg, eps, sp[0], 0, SAMPLE_THREADS);
    __syncthreads();
    // the walker's state
    double tot = g.prefix;
    uint64_t lastNz = base;
    unsigned k = g.begin;
    double rnd = srnd[k];
    for (int s = 0; s < nseg; ++s) {
        const double* cur = sp[s & 1];
        if (threadIdx.x >= 32) {
            if (s + 1 < nseg) {
                sample_stage(psi, base + (uint64_t)(s + 1) * seg, seg, eps, sp[(s + 1) & 1], 32, SAMPLE_THREADS - 32);
            }
        } else if (threadIdx.x == 0) {
            const uint64_t at = base + (uint64_t)s * seg;
            for (int i = 0; i < seg && k < end; i += SAMPLE_BATCH) {
                const int nb = (seg - i < SAMPLE_BATCH) ? seg - i : SAMPLE_BATCH;
                double p[SAMPLE_BATCH], t[SAMPLE_BATCH];
                double acc = tot;
#pragma unroll
                for (int j = 0; j < SAMPLE_BATCH; ++j) {
                    p[j] = (j < nb) ? cur[i + j] : 0.0;
                    acc = __dadd_rn(acc, p[j]);
                    t[j] = acc;
                }
                // tot only grows: if the batch's last tot does not serve shot k, no tot in the batch does
                if (acc > rnd || (1.0 - acc) <= fpEps) {
#pragma unroll
                    for (int j = 0; j < SAMPLE_BATCH; ++j) {
                        if (p[j] > 0.0) {
                            while (k < end && (t[j] > rnd || (1.0 - t[j]) <= fpEps)) {
                                keys[slot[k]] = at + i + j;
                                if (++k < end) {
                                    rnd = srnd[k];
                                }
                            }
                        }
                    }
                }
#pragma unroll
                for (int j = 0; j < SAMPLE_BATCH; ++j) {
                    if (p[j] > 0.0) {
                        lastNz = at + i + j;
                    }
                }
                tot = acc;
            }
        }
        if (__syncthreads_or(threadIdx.x == 0 && k == end)) { // every shot of the group is served
            break;
        }
    }
    if (threadIdx.x == 0) {
        for (; k < end; ++k) {
            keys[slot[k]] = lastNz;
        }
    }
    __syncthreads(); // the walker's picks are visible to the CTA
    if (!key.ident) {
        for (unsigned q = g.begin + threadIdx.x; q < end; q += SAMPLE_THREADS) {
            keys[slot[q]] = sample_key(keys[slot[q]], key);
        }
    }
}

// keys[i] = t(the search of rnds[i]) on a flushed state (the map was checked by the caller)
static int sample_keyed_impl(State* s, int n_shots, const double* rnds, const SampleKey& key, uint64_t* keys)
{
    const uint64_t n = s->dim();
    std::fill(keys, keys + n_shots, sample_key(n - 1U, key));
    if (!s->amps || !n_shots) {
        return B200SV_OK;
    }
    const uint64_t chunk = std::min<uint64_t>(n, 1ULL << 14);
    const uint64_t nchunks = n / chunk;
    SV_TRY(ensure_scratch(s, nchunks));
    const double eps = (s->prec == 32) ? 1.7763568394002505e-15 : 6.310887241768095e-30; // REAL1_EPSILON (qrack_types.hpp:206,209)
    const double fpEps = (s->prec == 32) ? 2.98023223876953125e-08 : 5.551115123125783e-17; // FP_NORM_EPSILON
    SV_TRY(with_prec(s, [&](auto r) {
        using R = decltype(r);
        k_chunk_sums<R><<<(unsigned)nchunks, 256, 0, s->stream>>>((const typename Cx<R>::type*)s->amps, chunk, (R)eps, s->d_scratch);
        return launched(s);
    }));
    SV_TRY(read_scratch(s, (int)nchunks));
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
    // shots in ascending rnd: a shot's chunk (the first c whose prefix[c + 1] exceeds rnd or comes within fpEps of 1, at
    // lastNonzeroChunk at the latest) never decreases with rnd, so one walk over the chunks assigns them all, and the shots of
    // a chunk come out contiguous and in ascending rnd, as the search wants them
    std::vector<std::pair<double, unsigned>> sorted((size_t)n_shots);
    for (int i = 0; i < n_shots; ++i) {
        sorted[(size_t)i] = {rnds[i], (unsigned)i};
    }
    std::sort(sorted.begin(), sorted.end());
    std::vector<SampleGroup> groups;
    uint64_t c = 0;
    for (int k = 0; k < n_shots; ++k) {
        const double rnd = sorted[(size_t)k].first;
        while (c < lastNonzeroChunk && !(prefix[c + 1] > rnd) && !((1.0 - prefix[c + 1]) <= fpEps)) {
            ++c;
        }
        if (groups.empty() || groups.back().c != c) {
            groups.push_back(SampleGroup{prefix[c], (unsigned)c, (unsigned)k});
        }
    }
    groups.push_back(SampleGroup{0.0, 0U, (unsigned)n_shots});
    // one device buffer: keys (by shot), rnds and slots (sorted), groups; staged through the pinned mirror of the scratch when
    // it fits there, else through pageable memory
    const size_t S = (size_t)n_shots;
    const size_t offRnd = S * sizeof(uint64_t), offSlot = offRnd + S * sizeof(double);
    const size_t offGroup = (offSlot + S * sizeof(unsigned) + 15) & ~(size_t)15;
    const size_t bytes = offGroup + groups.size() * sizeof(SampleGroup);
    DevBuf<> own;
    void* dev = nullptr;
    SV_TRY(scratch_or_own(s, 0, bytes, own, &dev));
    char* d = static_cast<char*>(dev);
    std::vector<char> pageable;
    char* h = reinterpret_cast<char*>(s->h_scratch);
    if (own) {
        pageable.resize(bytes);
        h = pageable.data();
    }
    double* hr = reinterpret_cast<double*>(h + offRnd);
    unsigned* hs = reinterpret_cast<unsigned*>(h + offSlot);
    for (size_t k = 0; k < S; ++k) {
        hr[k] = sorted[k].first;
        hs[k] = sorted[k].second;
    }
    memcpy(h + offGroup, groups.data(), groups.size() * sizeof(SampleGroup));
    SV_CUDA(cudaMemcpyAsync(d + offRnd, h + offRnd, bytes - offRnd, cudaMemcpyHostToDevice, s->stream));
    SV_TRY(with_prec(s, [&](auto r) {
        using R = decltype(r);
        k_sample_search<R><<<(unsigned)(groups.size() - 1), SAMPLE_THREADS, 0, s->stream>>>((const typename Cx<R>::type*)s->amps,
            chunk, eps, fpEps, reinterpret_cast<const SampleGroup*>(d + offGroup), reinterpret_cast<const double*>(d + offRnd),
            reinterpret_cast<const unsigned*>(d + offSlot), reinterpret_cast<unsigned long long*>(d), key);
        return launched(s);
    }));
    SV_CUDA(cudaMemcpyAsync(own ? (void*)keys : (void*)h, d, S * sizeof(uint64_t), cudaMemcpyDeviceToHost, s->stream));
    SV_CUDA(cudaStreamSynchronize(s->stream));
    if (!own) {
        memcpy(keys, h, S * sizeof(uint64_t));
    }
    return B200SV_OK;
}

} // namespace b200sv
