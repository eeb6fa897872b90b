// lossy.cuh — lossy state checkpoints (QInterface::LossySaveStateVector / LossyLoadStateVector): the reference's TurboQuant
// block codec (include/statevector_turboquant.hpp), bit-exact, with the rotations on the device.
//
// With D = 2^p, block k is amplitudes [kD, (k+1)D) read as the real vector v = [re_0, im_0, re_1, im_1, ..] of length d = 2D,
// which is exactly the block's interleaved amplitudes in memory (zero-padded when the state is shorter than one block).
//   rotation  R, d x d column-major, from the seed: d^2 draws of std::normal_distribution<real>(0, 1) over
//             std::mt19937_64(seed), then modified Gram-Schmidt (sequential sums, norm clamped at 1e-8).  Built on the host;
//             the library's host code is compiled without FP contraction, so it matches the reference's own code bit for bit.
//   encode    w_i = sum_j R[j d + i] v_j;  scale = sqrt(sum_j w_j^2 / d + 1e-8);  bucket = (int)((clamp(w, lo, hi - step) - lo)
//             / step) with lo = -3 scale, hi = 3 scale, step = (hi - lo) / 2^b (bucket 0 when step < 1e-8); bucket j's b bits
//             at bit j b of little-endian 64-bit words.
//   decode    u_j = lo + (bucket_j + 0.5) step;  out_i = sum_j R[i d + j] u_j.
// Every sum runs over j in order, and every multiply and add is a separate IEEE operation in `real` (__fmul_rn / __fadd_rn:
// no contraction, whatever the compile flags), so device files and decodes equal the reference's bit for bit.
//
// Kernels (one instantiation per precision and d = 4 .. 128, i.e. 1 <= p <= 6): a CTA stages the d x d matrix in shared
// memory once (64 KB fp32 / 128 KB fp64 at d = 128): R for the encode, R^T for the decode, so both products read it the
// same conflict-free way.  Each warp takes LOSSY_G * (32 / min(d, 32)) blocks at a time: the block vectors go to a
// warp-private shared buffer, each lane owns d / min(d, 32) consecutive outputs of LOSSY_G blocks and keeps one sequential
// chain per output, so every matrix element read from shared memory serves LOSSY_G blocks.  The encode then forms each
// block's scale (one lane per block, sequential), and one lane per 64-bit word assembles the word from the buckets that
// overlap it (OR, exact in any order).  Scales and words go to a device staging buffer; the host streams them to and from
// the file in chunks through pinned buffers of at most LOSSY_STAGE bytes, so no full-state host copy is ever made.
// Included by b200sv.cu (same translation unit as the other kernels).
#pragma once

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <random>
#include <vector>

namespace b200sv {

static const int LOSSY_THREADS = 256;
static const int LOSSY_WARPS = LOSSY_THREADS / 32;
static const int LOSSY_G = 4;                          // blocks per lane chain set: each shared R element serves LOSSY_G blocks
static const size_t LOSSY_STAGE = (size_t)64 << 20;   // staging bytes (scales + words) per chunk
static const size_t LOSSY_HEADER = 3 * sizeof(size_t); // capacity, BLOCK, num_blocks

// ---- separate IEEE operations in `real` (host: the library is built with -ffp-contract=off) ----------------------------
__host__ __device__ __forceinline__ float lq_add(float a, float b)
{
#ifdef __CUDA_ARCH__
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ __forceinline__ double lq_add(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ __forceinline__ float lq_mul(float a, float b)
{
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ __forceinline__ double lq_mul(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ __forceinline__ float lq_div(float a, float b)
{
#ifdef __CUDA_ARCH__
    return __fdiv_rn(a, b);
#else
    return a / b;
#endif
}
__host__ __device__ __forceinline__ double lq_div(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}
__host__ __device__ __forceinline__ float lq_sqrt(float a)
{
#ifdef __CUDA_ARCH__
    return __fsqrt_rn(a);
#else
    return std::sqrt(a);
#endif
}
__host__ __device__ __forceinline__ double lq_sqrt(double a)
{
#ifdef __CUDA_ARCH__
    return __dsqrt_rn(a);
#else
    return std::sqrt(a);
#endif
}

// the quantiser's range for one block: lo, step (hi - step is the upper clamp)
template <typename real> struct LqRange {
    real lo, hi, step;
    __host__ __device__ __forceinline__ LqRange(real scale, int bits)
    {
        lo = lq_mul((real)-3.0, scale);
        hi = lq_mul((real)3.0, scale);
        step = lq_div(lq_add(hi, -lo), (real)(1 << bits));
    }
    __host__ __device__ __forceinline__ int bucket(real w, int bits) const
    {
        if (step < (real)1e-8) {
            return 0;
        }
        const real top = lq_add(hi, -step);
        const real m = (w < top) ? w : top; // std::min(hi - step, w)
        const real c = (lo < m) ? m : lo;   // std::max(lo, m)
        int b = (int)lq_div(lq_add(c, -lo), step);
        const int levels = 1 << bits;
        return b < 0 ? 0 : (b >= levels ? levels - 1 : b);
    }
    __host__ __device__ __forceinline__ real dequant(int bucket) const
    {
        return lq_add(lo, lq_mul(lq_add((real)bucket, (real)0.5), step));
    }
};

template <typename real> __host__ __device__ __forceinline__ real lq_scale(real sumsq, int d)
{
    return lq_sqrt(lq_add(lq_div(sumsq, (real)d), (real)1e-8));
}

// bucket j of a block's packed words (a bucket may straddle two words)
__host__ __device__ __forceinline__ int lq_unpack(const unsigned long long* words, int j, int bits)
{
    const int off = j * bits, w = off >> 6, bit = off & 63;
    const unsigned long long m = (1ULL << bits) - 1U;
    unsigned long long v = (words[w] >> bit) & m;
    if (bit + bits > 64) {
        v |= (words[w + 1] << (64 - bit)) & m;
    }
    return (int)v;
}

// ---- host: the rotation ---------------------------------------------------------------------------------------------
template <typename real> static void lossy_rotation_host(int d, uint64_t seed, real* R)
{
    std::mt19937_64 rng(seed);
    std::normal_distribution<real> normal((real)0, (real)1);
    const size_t dd = (size_t)d * d;
    for (size_t t = 0; t < dd; ++t) {
        R[t] = normal(rng);
    }
    for (int j = 0; j < d; ++j) {
        real* cj = R + (size_t)j * d;
        real nrm = 0;
        for (int i = 0; i < d; ++i) {
            nrm = lq_add(nrm, lq_mul(cj[i], cj[i]));
        }
        nrm = lq_sqrt(nrm);
        if (nrm < (real)1e-8) {
            nrm = (real)1e-8;
        }
        for (int i = 0; i < d; ++i) {
            cj[i] = lq_div(cj[i], nrm);
        }
        for (int k = j + 1; k < d; ++k) {
            real* ck = R + (size_t)k * d;
            real dot = 0;
            for (int i = 0; i < d; ++i) {
                dot = lq_add(dot, lq_mul(cj[i], ck[i]));
            }
            for (int i = 0; i < d; ++i) {
                ck[i] = lq_add(ck[i], -lq_mul(dot, cj[i]));
            }
        }
    }
}

// ---- device -----------------------------------------------------------------------------------------------------------
template <int D2> struct LqShape {
    static const int LPB = D2 < 32 ? D2 : 32; // lanes per block
    static const int BPP = 32 / LPB;          // blocks side by side in a warp
    static const int K = D2 / LPB;            // consecutive outputs per lane
    static const int WB = BPP * LOSSY_G;      // blocks per warp batch
};

template <typename real, int D2> static size_t lossy_smem()
{
    return ((size_t)D2 * D2 + (size_t)LOSSY_WARPS * LqShape<D2>::WB * D2 + LOSSY_WARPS * LqShape<D2>::WB) * sizeof(real);
}

// out[blk][i] = sum_j M[j D2 + i] x[blk][j] for the warp's batch; x is V laid out [bsub][j][g], the result overwrites it
template <typename real, int D2> __device__ __forceinline__ void lq_rotate_batch(const real* M, real* V, int lane)
{
    typedef LqShape<D2> S;
    const int bsub = lane / S::LPB, i0 = (lane % S::LPB) * S::K;
    real acc[S::K][LOSSY_G];
#pragma unroll
    for (int k = 0; k < S::K; ++k) {
#pragma unroll
        for (int g = 0; g < LOSSY_G; ++g) {
            acc[k][g] = (real)0;
        }
    }
    const real* Vb = V + (size_t)bsub * D2 * LOSSY_G;
#pragma unroll 4
    for (int j = 0; j < D2; ++j) {
        real r[S::K], v[LOSSY_G];
#pragma unroll
        for (int k = 0; k < S::K; ++k) {
            r[k] = M[j * D2 + i0 + k];
        }
#pragma unroll
        for (int g = 0; g < LOSSY_G; ++g) {
            v[g] = Vb[j * LOSSY_G + g];
        }
#pragma unroll
        for (int k = 0; k < S::K; ++k) {
#pragma unroll
            for (int g = 0; g < LOSSY_G; ++g) {
                acc[k][g] = lq_add(acc[k][g], lq_mul(r[k], v[g]));
            }
        }
    }
    __syncwarp();
    real* Vo = V + (size_t)bsub * D2 * LOSSY_G;
#pragma unroll
    for (int k = 0; k < S::K; ++k) {
#pragma unroll
        for (int g = 0; g < LOSSY_G; ++g) {
            Vo[(i0 + k) * LOSSY_G + g] = acc[k][g];
        }
    }
    __syncwarp();
}

// V slot of (block in batch, coordinate j)
template <int D2> __device__ __forceinline__ int lq_slot(int blk, int j)
{
    return ((blk / LOSSY_G) * D2 + j) * LOSSY_G + (blk % LOSSY_G);
}

template <typename real> __device__ __forceinline__ void lq_stage_matrix(real* M, const real* Mg, int dd)
{
    for (int t = threadIdx.x; t < dd; t += blockDim.x) {
        M[t] = Mg[t];
    }
    __syncthreads();
}

// encode blocks [blk0, blk0 + nblk) of the state (nreal = 2 dim reals) into scales[0 .. nblk) and words[0 .. nblk * nwords)
template <typename real, int D2>
__global__ void __launch_bounds__(LOSSY_THREADS) k_lossy_encode(const real* __restrict__ amps, uint64_t nreal, uint64_t blk0,
    uint64_t nblk, const real* __restrict__ Rg, int bits, int nwords, real* __restrict__ scales,
    unsigned long long* __restrict__ words)
{
    typedef LqShape<D2> S;
    extern __shared__ __align__(16) unsigned char lq_smem[];
    real* M = (real*)lq_smem;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    real* V = M + D2 * D2 + (size_t)warp * S::WB * D2;
    real* SC = M + D2 * D2 + (size_t)LOSSY_WARPS * S::WB * D2 + warp * S::WB;
    lq_stage_matrix(M, Rg, D2 * D2);

    const uint64_t nbatch = (nblk + S::WB - 1) / S::WB;
    for (uint64_t bt = (uint64_t)blockIdx.x * LOSSY_WARPS + warp; bt < nbatch; bt += (uint64_t)gridDim.x * LOSSY_WARPS) {
        const uint64_t b0 = bt * S::WB;
        for (int t = lane; t < S::WB * D2; t += 32) {
            const int blk = t / D2, j = t % D2;
            const uint64_t gi = (blk0 + b0 + blk) * D2 + j;
            V[lq_slot<D2>(blk, j)] = (b0 + blk < nblk && gi < nreal) ? amps[gi] : (real)0;
        }
        __syncwarp();
        lq_rotate_batch<real, D2>(M, V, lane);
        if (lane < S::WB) {
            real sum = (real)0;
            for (int j = 0; j < D2; ++j) {
                const real w = V[lq_slot<D2>(lane, j)];
                sum = lq_add(sum, lq_mul(w, w));
            }
            const real sc = lq_scale(sum, D2);
            SC[lane] = sc;
            if (b0 + lane < nblk) {
                scales[b0 + lane] = sc;
            }
        }
        __syncwarp();
        for (int t = lane; t < S::WB * nwords; t += 32) {
            const int blk = t / nwords, w = t % nwords;
            if (b0 + blk >= nblk) {
                continue;
            }
            const LqRange<real> rg(SC[blk], bits);
            const int jlo = (64 * w) / bits, jhi = min(D2 - 1, (64 * w + 63) / bits);
            unsigned long long word = 0;
            for (int j = jlo; j <= jhi; ++j) {
                const unsigned long long bk = (unsigned long long)rg.bucket(V[lq_slot<D2>(blk, j)], bits);
                const int off = j * bits - 64 * w;
                word |= (off >= 0) ? (bk << off) : (bk >> -off);
            }
            words[(b0 + blk) * nwords + w] = word;
        }
        __syncwarp();
    }
}

// decode nblk blocks from staging into the state: block t of the launch is staging block cb = blist ? blist[t] : t, state
// block blk0 + cb
template <typename real, int D2>
__global__ void __launch_bounds__(LOSSY_THREADS) k_lossy_decode(real* __restrict__ amps, uint64_t nreal, uint64_t blk0,
    uint64_t nblk, const unsigned* __restrict__ blist, const real* __restrict__ RTg, int bits, int nwords,
    const real* __restrict__ scales, const unsigned long long* __restrict__ words)
{
    typedef LqShape<D2> S;
    extern __shared__ __align__(16) unsigned char lq_smem[];
    real* M = (real*)lq_smem;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    real* V = M + D2 * D2 + (size_t)warp * S::WB * D2;
    lq_stage_matrix(M, RTg, D2 * D2);

    const uint64_t nbatch = (nblk + S::WB - 1) / S::WB;
    for (uint64_t bt = (uint64_t)blockIdx.x * LOSSY_WARPS + warp; bt < nbatch; bt += (uint64_t)gridDim.x * LOSSY_WARPS) {
        const uint64_t b0 = bt * S::WB;
        for (int t = lane; t < S::WB * D2; t += 32) {
            const int blk = t / D2, j = t % D2;
            real u = (real)0;
            if (b0 + blk < nblk) {
                const uint64_t cb = blist ? (uint64_t)blist[b0 + blk] : b0 + blk;
                const LqRange<real> rg(scales[cb], bits);
                u = rg.dequant(lq_unpack(words + cb * nwords, j, bits));
            }
            V[lq_slot<D2>(blk, j)] = u;
        }
        __syncwarp();
        lq_rotate_batch<real, D2>(M, V, lane);
        for (int t = lane; t < S::WB * D2; t += 32) {
            const int blk = t / D2, i = t % D2;
            if (b0 + blk < nblk) {
                const uint64_t cb = blist ? (uint64_t)blist[b0 + blk] : b0 + blk;
                const uint64_t gi = (blk0 + cb) * D2 + i;
                if (gi < nreal) {
                    amps[gi] = V[lq_slot<D2>(blk, i)];
                }
            }
        }
        __syncwarp();
    }
}

template <typename real, int D2> static unsigned lossy_grid(State* s, uint64_t nblk, size_t smem)
{
    int per = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, k_lossy_encode<real, D2>, LOSSY_THREADS, smem);
    const uint64_t want = (nblk + (uint64_t)LOSSY_WARPS * LqShape<D2>::WB - 1) / ((uint64_t)LOSSY_WARPS * LqShape<D2>::WB);
    const uint64_t cap = (uint64_t)sm_count(s->dev) * (per > 0 ? per : 1);
    return (unsigned)std::max<uint64_t>(1, std::min(want, cap));
}

template <typename real, int D2>
static int lossy_launch_t(State* s, bool encode, uint64_t blk0, uint64_t nblk, const unsigned* blist, const real* M, int bits,
    int nwords, real* scales, unsigned long long* words)
{
    const size_t smem = lossy_smem<real, D2>();
    SV_CUDA(cudaFuncSetAttribute(k_lossy_encode<real, D2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    SV_CUDA(cudaFuncSetAttribute(k_lossy_decode<real, D2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const unsigned grid = lossy_grid<real, D2>(s, nblk, smem);
    const uint64_t nreal = 2 * s->dim();
    if (encode) {
        k_lossy_encode<real, D2><<<grid, LOSSY_THREADS, smem, s->stream>>>((const real*)s->amps, nreal, blk0, nblk, M, bits,
                                                                           nwords, scales, words);
    } else {
        k_lossy_decode<real, D2><<<grid, LOSSY_THREADS, smem, s->stream>>>((real*)s->amps, nreal, blk0, nblk, blist, M, bits,
                                                                           nwords, scales, words);
    }
    return launched(s);
}

template <typename real>
static int lossy_launch(State* s, bool encode, int p, uint64_t blk0, uint64_t nblk, const unsigned* blist, const real* M,
    int bits, int nwords, real* scales, unsigned long long* words)
{
    switch (p) {
    case 1: return lossy_launch_t<real, 4>(s, encode, blk0, nblk, blist, M, bits, nwords, scales, words);
    case 2: return lossy_launch_t<real, 8>(s, encode, blk0, nblk, blist, M, bits, nwords, scales, words);
    case 3: return lossy_launch_t<real, 16>(s, encode, blk0, nblk, blist, M, bits, nwords, scales, words);
    case 4: return lossy_launch_t<real, 32>(s, encode, blk0, nblk, blist, M, bits, nwords, scales, words);
    case 5: return lossy_launch_t<real, 64>(s, encode, blk0, nblk, blist, M, bits, nwords, scales, words);
    case 6: return lossy_launch_t<real, 128>(s, encode, blk0, nblk, blist, M, bits, nwords, scales, words);
    default: return einval("lossy: block power outside 1..6");
    }
}

static int lq_einval(const std::string& msg)
{
    return einval(msg.c_str());
}

// ---- host: file format ------------------------------------------------------------------------------------------------
// header: size_t capacity, size_t BLOCK, size_t num_blocks; then per block: size_t D, int BITS, bool initialized,
// uint64 seed, [real scale if initialized], size_t NWORDS, NWORDS x uint64
static inline size_t lossy_record_bytes(size_t real_bytes, int nwords)
{
    return sizeof(size_t) + sizeof(int) + sizeof(bool) + sizeof(uint64_t) + real_bytes + sizeof(size_t) + 8 * (size_t)nwords;
}

template <typename real>
static char* lossy_put_record(char* o, size_t D, int bits, uint64_t seed, real scale, int nwords, const unsigned long long* w)
{
    const bool init = true;
    const size_t nw = (size_t)nwords;
    memcpy(o, &D, sizeof(D));
    o += sizeof(D);
    memcpy(o, &bits, sizeof(bits));
    o += sizeof(bits);
    memcpy(o, &init, sizeof(init));
    o += sizeof(init);
    memcpy(o, &seed, sizeof(seed));
    o += sizeof(seed);
    memcpy(o, &scale, sizeof(scale));
    o += sizeof(scale);
    memcpy(o, &nw, sizeof(nw));
    o += sizeof(nw);
    memcpy(o, w, 8 * nw);
    return o + 8 * nw;
}

struct LqFile {
    FILE* f = nullptr;
    ~LqFile()
    {
        if (f) {
            fclose(f);
        }
    }
};

// device and pinned staging of one chunk, freed on every exit path
template <typename real> struct LqStage {
    DevBuf<real> d_scales;
    DevBuf<unsigned long long> d_words;
    DevBuf<real> d_mat;
    DevBuf<unsigned> d_list;
    PinnedBuf<real> h_scales;
    PinnedBuf<unsigned long long> h_words;
    PinnedBuf<unsigned> h_list;
    int alloc(size_t cb, int nwords, int d, bool lists)
    {
        SV_CUDA(cudaMalloc(&d_scales.p, cb * sizeof(real)));
        SV_CUDA(cudaMalloc(&d_words.p, cb * nwords * 8));
        SV_CUDA(cudaMalloc(&d_mat.p, (size_t)d * d * sizeof(real)));
        SV_CUDA(cudaMallocHost(&h_scales.p, cb * sizeof(real)));
        SV_CUDA(cudaMallocHost(&h_words.p, cb * nwords * 8));
        if (lists) {
            SV_CUDA(cudaMalloc(&d_list.p, cb * sizeof(unsigned)));
            SV_CUDA(cudaMallocHost(&h_list.p, cb * sizeof(unsigned)));
        }
        return B200SV_OK;
    }
};

static inline size_t lossy_chunk_blocks(size_t nblocks, size_t real_bytes, int nwords)
{
    const size_t cb = LOSSY_STAGE / (real_bytes + 8 * (size_t)nwords);
    return std::max<size_t>(1, std::min(nblocks, cb));
}

template <typename real> static int lossy_save_t(State* s, const char* path, int p, int bits, uint64_t seed)
{
    const size_t D = (size_t)1 << p, cap = s->dim(), nblocks = (cap + D - 1) / D;
    const int d = (int)(2 * D), nwords = (d * bits + 63) / 64;
    const size_t rec = lossy_record_bytes(sizeof(real), nwords);
    std::vector<real> R((size_t)d * d);
    lossy_rotation_host<real>(d, seed, R.data());

    LqFile lf;
    lf.f = fopen(path, "wb");
    if (!lf.f) {
        return lq_einval(std::string("lossy_save: cannot open '") + path + "' for writing");
    }
    const size_t hdr[3] = { cap, D, nblocks };
    bool ok = fwrite(hdr, sizeof(hdr), 1, lf.f) == 1;
    const size_t cb = lossy_chunk_blocks(nblocks, sizeof(real), nwords);
    std::vector<char> out(cb * rec);

    if (!s->amps) {
        // the zero state: every block is the zero block (w = 0, scale = sqrt(1e-8)), encoded once here and repeated
        const real sc = lq_scale((real)0, d);
        const LqRange<real> rg(sc, bits);
        std::vector<unsigned long long> w(nwords, 0ULL);
        const unsigned long long bk = (unsigned long long)rg.bucket((real)0, bits);
        for (int j = 0; j < d; ++j) {
            const int off = j * bits, wi = off >> 6, bit = off & 63;
            w[wi] |= bk << bit;
            if (bit + bits > 64) {
                w[wi + 1] |= bk >> (64 - bit);
            }
        }
        for (size_t t = 0; t < cb; ++t) {
            lossy_put_record<real>(out.data() + t * rec, D, bits, seed, sc, nwords, w.data());
        }
        for (size_t b0 = 0; ok && b0 < nblocks; b0 += cb) {
            const size_t nb = std::min(cb, nblocks - b0);
            ok = fwrite(out.data(), rec, nb, lf.f) == nb;
        }
    } else {
        LqStage<real> st;
        SV_TRY(st.alloc(cb, nwords, d, false));
        SV_CUDA(cudaMemcpyAsync(st.d_mat, R.data(), R.size() * sizeof(real), cudaMemcpyHostToDevice, s->stream));
        for (size_t b0 = 0; ok && b0 < nblocks; b0 += cb) {
            const size_t nb = std::min(cb, nblocks - b0);
            SV_TRY(lossy_launch<real>(s, true, p, b0, nb, nullptr, st.d_mat, bits, nwords, st.d_scales, st.d_words));
            SV_CUDA(cudaMemcpyAsync(st.h_scales, st.d_scales, nb * sizeof(real), cudaMemcpyDeviceToHost, s->stream));
            SV_CUDA(cudaMemcpyAsync(st.h_words, st.d_words, nb * nwords * 8, cudaMemcpyDeviceToHost, s->stream));
            SV_CUDA(cudaStreamSynchronize(s->stream));
            char* o = out.data();
            for (size_t t = 0; t < nb; ++t) {
                o = lossy_put_record<real>(o, D, bits, seed, st.h_scales[t], nwords, st.h_words + t * nwords);
            }
            ok = fwrite(out.data(), rec, nb, lf.f) == nb;
        }
    }
    const int closed = fclose(lf.f);
    lf.f = nullptr;
    if (!ok || closed) {
        return lq_einval(std::string("lossy_save: write to '") + path + "' failed");
    }
    return B200SV_OK;
}

// buffered sequential reader
struct LqReader {
    FILE* f;
    std::vector<char> buf;
    size_t pos = 0, len = 0;
    explicit LqReader(FILE* f_) : f(f_), buf((size_t)16 << 20) {}
    bool get(void* dst, size_t n)
    {
        char* o = (char*)dst;
        while (n) {
            if (pos == len) {
                len = fread(buf.data(), 1, buf.size(), f);
                pos = 0;
                if (!len) {
                    return false;
                }
            }
            const size_t m = std::min(n, len - pos);
            memcpy(o, buf.data() + pos, m);
            pos += m;
            o += m;
            n -= m;
        }
        return true;
    }
    bool at_end()
    {
        char c;
        return !get(&c, 1);
    }
};

struct LqGeometry {
    size_t cap, D, nblocks;
    int nq, p, bits;
};

static inline int lq_log2(size_t x)
{
    int l = 0;
    while (((size_t)1 << l) < x) {
        ++l;
    }
    return l;
}

// header and the first record's D / BITS / NWORDS (the reader is left after the header)
static int lossy_read_geometry(LqReader& rd, LqGeometry* g, long fsize)
{
    size_t hdr[3];
    if (!rd.get(hdr, sizeof(hdr))) {
        return einval("lossy: file is shorter than its header");
    }
    g->cap = hdr[0];
    g->D = hdr[1];
    g->nblocks = hdr[2];
    if (!g->cap || (g->cap & (g->cap - 1)) || g->cap > ((size_t)1 << 62)) {
        return einval("lossy: capacity is not a power of two");
    }
    if (!g->D || (g->D & (g->D - 1)) || g->D > ((size_t)1 << 30)) {
        return einval("lossy: BLOCK is not a power of two");
    }
    if (g->nblocks != (g->cap + g->D - 1) / g->D) {
        return einval("lossy: num_blocks does not match capacity / BLOCK");
    }
    g->nq = lq_log2(g->cap);
    g->p = lq_log2(g->D);
    // first record, read from a copy of the stream position
    char first[sizeof(size_t) + sizeof(int)];
    if (fsize < (long)(LOSSY_HEADER + sizeof(first))) {
        return einval("lossy: file has no block record");
    }
    memcpy(first, rd.buf.data() + rd.pos, std::min(sizeof(first), rd.len - rd.pos));
    size_t D;
    memcpy(&D, first, sizeof(D));
    memcpy(&g->bits, first + sizeof(D), sizeof(int));
    if (D != g->D) {
        return einval("lossy: a block's D differs from BLOCK");
    }
    return B200SV_OK;
}

static long lq_file_size(FILE* f)
{
    if (fseek(f, 0, SEEK_END)) {
        return -1;
    }
    const long n = ftell(f);
    rewind(f);
    return n;
}

// one record into (scale, words); `seed` out
template <typename real>
static int lossy_get_record(LqReader& rd, const LqGeometry& g, int nwords, real* scale, unsigned long long* words,
    uint64_t* seed)
{
    size_t D, nw;
    int bits;
    bool init;
    if (!rd.get(&D, sizeof(D)) || !rd.get(&bits, sizeof(bits)) || !rd.get(&init, sizeof(init)) || !rd.get(seed, sizeof(*seed))) {
        return einval("lossy: file ends inside a block record");
    }
    if (D != g.D) {
        return einval("lossy: a block's D differs from BLOCK");
    }
    if (bits != g.bits) {
        return einval("lossy: BITS differs between blocks");
    }
    *scale = (real)1;
    if (init && !rd.get(scale, sizeof(real))) {
        return einval("lossy: file ends inside a block record");
    }
    if (!rd.get(&nw, sizeof(nw))) {
        return einval("lossy: file ends inside a block record");
    }
    if (nw != (size_t)nwords) {
        return einval("lossy: NWORDS does not match (2 D BITS + 63) / 64 (is the file of the other precision?)");
    }
    if (!rd.get(words, 8 * nw)) {
        return einval("lossy: file ends inside a block record");
    }
    return B200SV_OK;
}

static int lossy_probe_impl(const char* path, int precision, int* nq, int* p, int* bits)
{
    LqFile lf;
    lf.f = fopen(path, "rb");
    if (!lf.f) {
        return lq_einval(std::string("lossy_probe: cannot open '") + path + "'");
    }
    const long fsize = lq_file_size(lf.f);
    LqReader rd(lf.f);
    LqGeometry g;
    const size_t rb = precision == 32 ? 4 : 8;
    SV_TRY(lossy_read_geometry(rd, &g, fsize));
    if (g.bits >= 1 && g.bits <= 30) {
        // the first record's NWORDS in this precision (an initialized record; an uninitialized one has no scale)
        const int nwords = (int)((2 * g.D * (size_t)g.bits + 63) / 64);
        size_t D, nw;
        int b;
        bool init;
        uint64_t seed;
        double sc;
        if (!rd.get(&D, sizeof(D)) || !rd.get(&b, sizeof(b)) || !rd.get(&init, sizeof(init)) || !rd.get(&seed, sizeof(seed)) ||
            (init && !rd.get(&sc, rb)) || !rd.get(&nw, sizeof(nw))) {
            return einval("lossy_probe: file ends inside the first block record");
        }
        if (nw != (size_t)nwords) {
            return einval("lossy_probe: NWORDS does not match (2 D BITS + 63) / 64 (is the file of the other precision?)");
        }
    }
    *nq = g.nq;
    *p = g.p;
    *bits = g.bits;
    return B200SV_OK;
}

template <typename real> static int lossy_load_t(State* s, const char* path)
{
    LqFile lf;
    lf.f = fopen(path, "rb");
    if (!lf.f) {
        return lq_einval(std::string("lossy_load: cannot open '") + path + "'");
    }
    const long fsize = lq_file_size(lf.f);
    LqReader rd(lf.f);
    LqGeometry g;
    SV_TRY(lossy_read_geometry(rd, &g, fsize));
    if (g.nq != s->nq) {
        return einval("lossy_load: the file's qubit count differs from the state's");
    }
    if (g.p < 1 || g.p > 6) {
        return einval("lossy_load: block power outside the device range 1..6");
    }
    if (g.bits < 1 || g.bits > 16) {
        return einval("lossy_load: BITS outside 1..16");
    }
    const int d = (int)(2 * g.D), nwords = (d * g.bits + 63) / 64;
    // every record is `rec` bytes, or sizeof(real) less when it is not initialized
    const size_t rec = lossy_record_bytes(sizeof(real), nwords);
    const size_t full = LOSSY_HEADER + g.nblocks * rec, least = LOSSY_HEADER + g.nblocks * (rec - sizeof(real));
    if (fsize < 0 || (size_t)fsize > full || (size_t)fsize < least || (full - (size_t)fsize) % sizeof(real)) {
        return einval("lossy_load: file length does not match the state's precision and geometry");
    }

    const size_t cb = lossy_chunk_blocks(g.nblocks, sizeof(real), nwords);
    LqStage<real> st;
    SV_TRY(st.alloc(cb, nwords, d, true));
    std::map<uint64_t, int> seeds; // seed -> rotation index, in order of first appearance
    std::vector<std::vector<real>> rots; // R^T per rotation index
    std::vector<int> ridx(cb);
    int uploaded = -1;
    bool touched = false;
    int rc = B200SV_OK;
    for (size_t b0 = 0; b0 < g.nblocks && rc == B200SV_OK; b0 += cb) {
        const size_t nb = std::min(cb, g.nblocks - b0);
        std::vector<int> present;
        for (size_t t = 0; t < nb && rc == B200SV_OK; ++t) {
            uint64_t seed;
            rc = lossy_get_record<real>(rd, g, nwords, st.h_scales + t, st.h_words + t * nwords, &seed);
            if (rc != B200SV_OK) {
                break;
            }
            auto it = seeds.find(seed);
            if (it == seeds.end()) {
                it = seeds.emplace(seed, (int)rots.size()).first;
                std::vector<real> R((size_t)d * d), RT((size_t)d * d);
                lossy_rotation_host<real>(d, seed, R.data());
                for (int i = 0; i < d; ++i) {
                    for (int j = 0; j < d; ++j) {
                        RT[(size_t)j * d + i] = R[(size_t)i * d + j];
                    }
                }
                rots.push_back(std::move(RT));
            }
            ridx[t] = it->second;
            if (std::find(present.begin(), present.end(), it->second) == present.end()) {
                present.push_back(it->second);
            }
        }
        if (rc == B200SV_OK && b0 + nb == g.nblocks && !rd.at_end()) {
            rc = einval("lossy_load: trailing bytes after the last block record");
        }
        if (rc != B200SV_OK) {
            break;
        }
        if (!touched) {
            drop_pending(s);
            rc = alloc_amps(s, false);
            if (rc != B200SV_OK) {
                return rc;
            }
            touched = true;
        }
        SV_CUDA(cudaMemcpyAsync(st.d_scales, st.h_scales, nb * sizeof(real), cudaMemcpyHostToDevice, s->stream));
        SV_CUDA(cudaMemcpyAsync(st.d_words, st.h_words, nb * nwords * 8, cudaMemcpyHostToDevice, s->stream));
        // one launch per rotation present in the chunk (a file the reference writes has one seed: one launch, no list)
        for (const int r : present) {
            if (r != uploaded) {
                SV_CUDA(cudaMemcpyAsync(st.d_mat, rots[r].data(), rots[r].size() * sizeof(real), cudaMemcpyHostToDevice,
                                        s->stream));
                uploaded = r;
            }
            const unsigned* list = nullptr;
            size_t nl = nb;
            if (present.size() > 1) {
                nl = 0;
                for (size_t t = 0; t < nb; ++t) {
                    if (ridx[t] == r) {
                        st.h_list[nl++] = (unsigned)t;
                    }
                }
                SV_CUDA(cudaMemcpyAsync(st.d_list, st.h_list, nl * sizeof(unsigned), cudaMemcpyHostToDevice, s->stream));
                list = st.d_list;
            }
            SV_TRY(lossy_launch<real>(s, false, g.p, b0, nl, list, st.d_mat, g.bits, nwords, st.d_scales, st.d_words));
            if (list) {
                SV_CUDA(cudaStreamSynchronize(s->stream)); // h_list is rewritten for the next rotation
            }
        }
        SV_CUDA(cudaStreamSynchronize(s->stream)); // the pinned buffers are refilled for the next chunk
    }
    if (rc != B200SV_OK && touched) {
        // a record past the first chunk was malformed after part of the state was overwritten: leave the zero state
        if (s->external) {
            SV_CUDA(cudaMemsetAsync(s->amps, 0, (size_t)s->dim() * s->amp_bytes(), s->stream));
        } else {
            free_amps(s);
        }
    }
    return rc;
}

} // namespace b200sv
