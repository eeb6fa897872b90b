// rdm.cuh — the reduced density matrix (GetReducedDensityMatrix, reference src/qinterface/qinterface.cpp:886-944) as one
// read-only Gram sweep.
//
// With K the kept qubits and E the others (ascending), A[i][e] = psi[dep_K(i) | dep_E(e)] and rho = A A^H.  The reference
// asks GetAmplitude for every environment state and every pair of kept states, 2^n (1 + 2^k) device round trips.  Here:
//   * rows are indexed in ASCENDING kept-qubit order (row bit b = the b-th smallest kept qubit; the host permutes to the
//     caller's order), so that with qubit 0 kept the two amplitudes of an fp32 16-byte chunk are rows 2r and 2r + 1 of one
//     column, whatever position qubit 0 has in the caller's list;
//   * column e deposits its bits on the env qubits from low to high, so consecutive columns are contiguous memory whenever the
//     low qubits are env qubits (with qubit 0 env an fp32 chunk is columns 2c and 2c + 1 of one row);
//   * each CTA computes one D x D tile (I, J), I <= J, of rho (D = min(2^k, RDM_T)) over a share of the environment: it stages
//     slabs of RDM_SLAB / D columns of A's row blocks I and J in shared memory (as double2; 16-byte global loads), and each
//     thread accumulates an RB x RB block of the tile, every product and sum in double (an fp32 amplitude converted to double
//     makes each product exact; only the additions round);
//   * k <= log2 RDM_T is one tile and the environment is split across the CTAs, so the state is read once;
//   * per-CTA partials go into the double output with one atomic per tile entry and CTA.  The lower triangle is mirrored on
//     the host as conjugates, the diagonal's imaginary part set to exactly 0.
// Included by b200sv.cu (same translation unit as the other kernels).
#pragma once

#include <algorithm>
#include <vector>

namespace b200sv {

static const int RDM_T = 64;      // tile side (rows of rho per tile)
static const int RDM_SLAB = 1024; // amplitudes of one row block staged per slab: RDM_SLAB / D columns
static const int RDM_THREADS = 256;

struct RdmArgs {
    int k;              // kept qubits, ascending in kept[0..k-1]
    int kept[B200SV_RDM_MAX_QUBITS];
    uint64_t keptLow[B200SV_RDM_MAX_QUBITS]; // 2^kept[b] - 1, ascending (push_apart inserts a zero bit at each kept qubit)
    int logD;           // tile side D = 2^logD
    int nt;             // tiles per side: 2^k / D
    uint64_t cols;      // 2^(n - k) environment states
    uint64_t slabs;     // ceil(cols / (RDM_SLAB / D))
    int rowsFast;       // qubit 0 kept: consecutive load units walk rows (fp32: a chunk = rows 2r, 2r + 1)
};

// env column -> amplitude index bits (zero bits inserted at the kept qubits)
__device__ __forceinline__ uint64_t rdm_col(uint64_t e, const RdmArgs& a)
{
    for (int b = 0; b < a.k; ++b) {
        const uint64_t lo = e & a.keptLow[b];
        e = ((e ^ lo) << 1) | lo;
    }
    return e;
}

// stage the D rows of nb row blocks (block b: offsets rowOff[b D ..], into sm[b RDM_SLAB + c D + r], as double2) at columns
// col0 .. col0 + S - 1.  Load units: fp32 (rows 2r, 2r + 1; column c) when qubit 0 is kept, else (row r; columns 2c, 2c + 1);
// fp64 (row r; column c).  D S = RDM_SLAB, so every thread has the same fixed number of units per block, and all of its 16-byte
// loads of the slab are issued before the first is converted and stored.
template <typename R>
__device__ __forceinline__ void rdm_stage(const void* __restrict__ amps, const uint64_t* rowOff, uint64_t col0, const RdmArgs& a,
    int D, int S, int nb, double2* sm)
{
    constexpr bool F32 = sizeof(R) == 4;
    typedef typename std::conditional<F32, float4, double2>::type V;
    constexpr int UPT = (F32 ? RDM_SLAB / 2 : RDM_SLAB) / RDM_THREADS; // units per thread and block
    const V* __restrict__ p = reinterpret_cast<const V*>(amps);
    const bool pairRows = F32 && a.rowsFast, pairCols = F32 && !a.rowsFast;
    const int nr = pairRows ? (D >> 1) : D, nc = pairCols ? (S >> 1) : S;
    V v[2][UPT];
    int rr[UPT], cc[UPT];
#pragma unroll
    for (int x = 0; x < UPT; ++x) {
        const int u = threadIdx.x + x * RDM_THREADS;
        const int ur = a.rowsFast ? (u % nr) : (u / nc), uc = a.rowsFast ? (u / nr) : (u % nc);
        rr[x] = pairRows ? 2 * ur : ur;
        cc[x] = pairCols ? 2 * uc : uc;
        const bool ok = col0 + (uint64_t)cc[x] < a.cols;
        const uint64_t col = ok ? rdm_col(col0 + (uint64_t)cc[x], a) : 0U;
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            v[b][x] = V{};
            if (ok && b < nb) {
                v[b][x] = p[(rowOff[b * D + rr[x]] | col) >> (F32 ? 1 : 0)];
            }
        }
    }
#pragma unroll
    for (int x = 0; x < UPT; ++x) {
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            if (b < nb) {
                double2* o = sm + b * RDM_SLAB;
                if constexpr (F32) {
                    o[cc[x] * D + rr[x]] = make_double2((double)v[b][x].x, (double)v[b][x].y);
                    o[pairRows ? (cc[x] * D + rr[x] + 1) : ((cc[x] + 1) * D + rr[x])] =
                        make_double2((double)v[b][x].z, (double)v[b][x].w);
                } else {
                    o[cc[x] * D + rr[x]] = v[b][x];
                }
            }
        }
    }
}

// out[(i << k) + j] (interleaved re, im; internal ascending row order) += sum_e A[i][e] conj(A[j][e]) for the tiles I <= J.
// grid = (upper-triangle tiles, environment splits); RB = the side of each thread's register block (min(4, D)).
template <typename R, int RB>
__global__ void __launch_bounds__(RDM_THREADS, 2) k_rdm(const void* __restrict__ amps, RdmArgs a, double* out)
{
    extern __shared__ __align__(16) unsigned char rdmSmem[];
    const int D = 1 << a.logD, S = RDM_SLAB >> a.logD;
    const int TPS = D / RB;                      // threads per tile side
    const int TPT = TPS * TPS;                   // threads per tile
    const int G = RDM_THREADS / TPT;             // column groups
    const int g = threadIdx.x / TPT, tl = threadIdx.x % TPT;
    const int tr = tl / TPS, tc = tl % TPS;

    // linear upper-triangle tile index -> (I, J), I <= J
    int t = blockIdx.x, I = 0;
    while (t >= a.nt - I) {
        t -= a.nt - I;
        ++I;
    }
    const int J = I + t;
    const bool diag = I == J;

    double2* sA = reinterpret_cast<double2*>(rdmSmem);
    double2* sB = diag ? sA : sA + RDM_SLAB;
    uint64_t* rowOff = reinterpret_cast<uint64_t*>(rdmSmem + 2 * RDM_SLAB * sizeof(double2)); // [0, D): block I, [D, 2D): J
    for (int r = threadIdx.x; r < 2 * D; r += RDM_THREADS) {
        const uint64_t row = (uint64_t)((r < D) ? I : J) * (uint64_t)D + (uint64_t)(r & (D - 1));
        uint64_t off = 0;
        for (int b = 0; b < a.k; ++b) {
            off |= ((row >> b) & 1U) << a.kept[b];
        }
        rowOff[r] = off;
    }

    double2 acc[RB][RB];
#pragma unroll
    for (int x = 0; x < RB; ++x) {
#pragma unroll
        for (int y = 0; y < RB; ++y) {
            acc[x][y] = make_double2(0.0, 0.0);
        }
    }
    for (uint64_t slab = blockIdx.y; slab < a.slabs; slab += gridDim.y) {
        __syncthreads(); // rowOff written / the previous slab consumed
        const uint64_t col0 = slab * (uint64_t)S;
        rdm_stage<R>(amps, rowOff, col0, a, D, S, diag ? 1 : 2, sA);
        __syncthreads();
        for (int c = g; c < S; c += G) {
            double2 u[RB], v[RB];
#pragma unroll
            for (int x = 0; x < RB; ++x) {
                u[x] = sA[c * D + tr + x * TPS];
                v[x] = sB[c * D + tc + x * TPS];
            }
#pragma unroll
            for (int x = 0; x < RB; ++x) {
#pragma unroll
                for (int y = 0; y < RB; ++y) {
                    // u conj(v)
                    acc[x][y].x = fma(u[x].x, v[y].x, fma(u[x].y, v[y].y, acc[x][y].x));
                    acc[x][y].y = fma(u[x].y, v[y].x, fma(-u[x].x, v[y].y, acc[x][y].y));
                }
            }
        }
    }

    const int rowBase = I * D, colBase = J * D, side = D * a.nt;
    if (G == 1) {
        // each entry of the tile belongs to one thread: one atomic per entry
#pragma unroll
        for (int x = 0; x < RB; ++x) {
#pragma unroll
            for (int y = 0; y < RB; ++y) {
                double* o = out + 2 * ((size_t)(rowBase + tr + x * TPS) * side + (colBase + tc + y * TPS));
                atomicAdd(o, acc[x][y].x);
                atomicAdd(o + 1, acc[x][y].y);
            }
        }
        return;
    }
    // several column groups hold partials of the same entries: fold the groups inside each warp with shuffles, then the warps
    // one after another into shared memory, then one atomic per entry
#pragma unroll
    for (int x = 0; x < RB; ++x) {
#pragma unroll
        for (int y = 0; y < RB; ++y) {
            for (int o = 16; o >= TPT; o >>= 1) {
                acc[x][y].x += __shfl_xor_sync(0xffffffffu, acc[x][y].x, o);
                acc[x][y].y += __shfl_xor_sync(0xffffffffu, acc[x][y].y, o);
            }
        }
    }
    __syncthreads(); // the slabs are no longer read
    double2* red = sA; // D * D <= RDM_SLAB entries when G > 1
    for (int e = threadIdx.x; e < D * D; e += RDM_THREADS) {
        red[e] = make_double2(0.0, 0.0);
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int w = 0; w < RDM_THREADS / 32; ++w) {
        __syncthreads();
        if (warp == w && (TPT >= 32 || lane < TPT)) {
#pragma unroll
            for (int x = 0; x < RB; ++x) {
#pragma unroll
                for (int y = 0; y < RB; ++y) {
                    double2& r = red[(tr + x * TPS) * D + tc + y * TPS];
                    r.x += acc[x][y].x;
                    r.y += acc[x][y].y;
                }
            }
        }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < D * D; e += RDM_THREADS) {
        double* o = out + 2 * ((size_t)(rowBase + e / D) * side + (colBase + e % D));
        atomicAdd(o, red[e].x);
        atomicAdd(o + 1, red[e].y);
    }
}

// One RDM sweep (arguments validated; the state is non-zero and flushed; 1 <= n).  out: 2 * 4^k doubles, caller's order.
static int launch_rdm(State* s, int k, const int* qubits, double* out)
{
    RdmArgs a{};
    a.k = k;
    std::vector<int> sorted(qubits, qubits + k);
    std::sort(sorted.begin(), sorted.end());
    for (int b = 0; b < k; ++b) {
        a.kept[b] = sorted[b];
        a.keptLow[b] = (1ULL << sorted[b]) - 1U;
    }
    a.logD = std::min(k, 6);
    const int D = 1 << a.logD, S = RDM_SLAB / D;
    a.nt = 1 << (k - a.logD);
    a.cols = 1ULL << (s->nq - k);
    a.slabs = (a.cols + S - 1) / S;
    a.rowsFast = (k > 0 && sorted[0] == 0) ? 1 : 0;
    const size_t shm = 2 * RDM_SLAB * sizeof(double2) + 2 * D * sizeof(uint64_t);
    const uint64_t tiles = (uint64_t)a.nt * (a.nt + 1) / 2;
    const int sms = sm_count(s->dev);
    const size_t dim = (size_t)1 << k;
    const size_t words = 2 * dim * dim;
    // the device sum: the state's scratch up to 1 MiB (k <= 8), else a buffer for this call only
    DevBuf<> own;
    void* dOut = nullptr;
    SV_TRY(scratch_or_own(s, 0, words * sizeof(double), own, &dOut));
    std::vector<double> host;
    if (own) {
        host.resize(words);
    }
    double* h = own ? host.data() : s->h_scratch;
    SV_TRY(with_prec(s, [&](auto r) {
        using R = decltype(r);
        void (*kern)(const void*, RdmArgs, double*) = (D >= 4) ? k_rdm<R, 4> : (D == 2) ? k_rdm<R, 2> : k_rdm<R, 1>;
        // one tile: the environment split over every CTA that fits on the device at once, so the state is read once at full
        // occupancy; several tiles: at least 2 x SMs CTAs in all
        int perSm = 2;
        SV_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, kern, RDM_THREADS, shm));
        const uint64_t want = (tiles == 1) ? (uint64_t)sms * std::max(perSm, 1) : (2U * sms + tiles - 1) / tiles;
        const unsigned splits = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(want, a.slabs));
        SV_CUDA(cudaMemsetAsync(dOut, 0, words * sizeof(double), s->stream));
        kern<<<dim3((unsigned)tiles, splits), RDM_THREADS, shm, s->stream>>>(s->amps, a, (double*)dOut);
        return launched(s);
    }));
    SV_CUDA(cudaMemcpyAsync(h, dOut, words * sizeof(double), cudaMemcpyDeviceToHost, s->stream));
    SV_CUDA(cudaStreamSynchronize(s->stream));

    // internal row index (bit b = sorted[b]) -> caller's index (bit p = qubits[p])
    std::vector<size_t> pos(dim);
    for (size_t i = 0; i < dim; ++i) {
        size_t p = 0;
        for (int b = 0; b < k; ++b) {
            if ((i >> b) & 1U) {
                p |= (size_t)1 << (std::find(qubits, qubits + k, sorted[b]) - qubits);
            }
        }
        pos[i] = p;
    }
    // only tiles I <= J were computed; every entry below the diagonal is the conjugate of its mirror, the diagonal is real
    for (size_t i = 0; i < dim; ++i) {
        double* row = out + 2 * pos[i] * dim;
        for (size_t j = 0; j < dim; ++j) {
            double re, im;
            if (i < j) {
                re = h[2 * (i * dim + j)];
                im = h[2 * (i * dim + j) + 1];
            } else if (i > j) {
                re = h[2 * (j * dim + i)];
                im = -h[2 * (j * dim + i) + 1];
            } else {
                re = h[2 * (i * dim + i)];
                im = 0.0;
            }
            row[2 * pos[j]] = re;
            row[2 * pos[j] + 1] = im;
        }
    }
    return B200SV_OK;
}

} // namespace b200sv
