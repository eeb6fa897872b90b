// fused.cu — the fused multi-gate sweep: a window of queued single-/controlled-single-qubit gates is applied in ONE
// pass over HBM (read 2^n amplitudes once, write once), instead of one read+write sweep per gate as in the reference
// (src/qengine/state.cpp:392-533 does one par_for_mask sweep per Apply2x2; src/qengine/cuda.cu:857-1059 one launch).
//
// Shape of one sweep (see DESIGN.md §K1-fused):
//   * tile  = 2^KC 16-byte chunks (64 KB) living in shared memory.  Its index bits are the low L qubits (so every
//     global access is a >= 2^L-amplitude contiguous run) plus up to H arbitrary "high" qubits chosen by the scheduler.
//   * passes: each pass picks RB "register" chunk bits; every thread holds a 2^RB-chunk sub-block in registers
//             (fp32: +qubit 0 inside the chunk) and applies every queued gate whose target is one of those bits (controls
//             anywhere: tile-local bits become a per-amplitude predicate, outside bits a per-tile predicate).  Diagonal
//             gates are index-only and ride along in any pass, on any qubit.
//   * data  : the first pass reads its sub-blocks straight from HBM and the last one writes straight back (128-bit
//             streaming accesses); between passes the sub-blocks are handed over through the tile in shared memory, in an
//             XOR-swizzled layout that keeps the butterflies bank-conflict free for any choice of register bits.
// The host-side scheduler below reorders only gates that commute (disjoint qubits, or shared qubits used diagonally by
// both) and never changes the product of the gate sequence.
#include "sv_common.cuh"

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>

namespace b200sv {

// the one kernel shape (DESIGN.md §7): a tile of 2^12 16-byte chunks, 256 threads, 2^4 register chunks per thread, 2 CTAs
// per SM
constexpr int FUSED_KC = 12;
constexpr int FUSED_NT = 256;
constexpr int FUSED_RB = 4;
constexpr int FUSED_MINB = 2;
constexpr int FUSED_L = 6; // low (contiguous) amplitude bits of a tile, both precisions

constexpr int MAX_HIGH = 8;
constexpr int MAX_PASS = 8;
constexpr int MAX_OPS = 96;
constexpr int MAX_HOST_OPS = 384; // gates per sweep before merging (LAYER / DIAG groups shrink them to <= MAX_OPS device ops)
constexpr int MAX_SLOTS = 128; // per-tile phase table (1 + register-bit phases of the DIAG ops); filled by warps 4..7
constexpr int MAX_NCH = 16; // register chunks per sub-block (RB <= 4)
constexpr int MAX_NA = 32;  // register amplitudes per sub-block
constexpr int MAX_JR = 6;   // register-bit indices the STAGE header has room for (5 are used)

// device op codes.  Single-gate ops: kind * 5 + jr (jr = register-bit index of the target; dense so that the dispatch is a
// shallow branch tree).  OPC_STAGE = per-bit phases + Hadamard butterflies; OPC_SCALE = per-tile scalar.
// bit 8 = the op has a sub-block predicate.
enum { K_XSWAP = 0, K_GEN_U = 1, K_GEN_P = 2 };
constexpr uint32_t OPC_PHGEN = 15U; // phase on the register amplitudes selected by emask (any register-bit predicate)
constexpr uint32_t OPC_SCALE = 16U; // multiply every amplitude by the per-tile scalar (outer phases x Hadamard scale)
// OPC_STAGE (r2): for every register bit J, in this order: [phase on the bit-J=1 half] then [Hadamard butterfly on J].
//   The phase of bit J is the product of (a) one per-tile table slot (members whose predicate is outer qubits AND bit J) and
//   (b) thread-level members (predicate: outer qubits AND thread bits AND bit J), tested per thread against the per-tile
//   "effective" (mask, val) table.  Group 0 = members without a register bit (thread-uniform phase on the whole sub-block).
//   header: emask = hmask | slotMask << 6 | anyMembers << 12 | activeBits << 13 | rotMask << 19 (bit J: the butterfly of bit J is a
//   real rotation [[c,-s],[s,c]] with (c, s) from the rotation table instead of a Hadamard); lmaskSb = first table slot;
//   lvalSb = first member | first rotation << 16; m[0] (as uint32) = seven 4-bit member counts (group 0, then register bits 0..5).
constexpr uint32_t OPC_STAGE = 17U;
// OPC_PH2 + pair: phase on the 2^(J-2)... register amplitudes that have BOTH register bits of the pair set (CZ / CPhase whose
// two qubits are register-resident); pair index = k * (k - 1) / 2 + j for bits j < k.
constexpr uint32_t OPC_PH2 = 18U; // .. 32 (15 pairs of 6 register bits)
// STAGE header fields (DevOp.emask) and member-count packing (first word of DevOp.m): 6-bit masks, 7 groups x 4 bits
constexpr int ST_SM_SHIFT = 6, ST_ANY_BIT = 12, ST_ACT_SHIFT = 13, ST_RM_SHIFT = 19, ST_CNT_BITS = 4;
constexpr uint32_t ST_MASK = 63U, ST_CNT_MASK = 15U;
constexpr uint32_t CODE_HAS_SB = 0x100U;
constexpr uint32_t CODE_HAS_OUTER = 0x200U; // the op has a predicate on qubits outside the tile: consult the per-tile ballot
constexpr int MAX_MEMBERS = 320; // thread-level phase members per sweep (8 bytes each in the double-buffered per-tile table)
// host (scheduler) op kinds
enum { OP_GENERAL = 0, OP_HAD = 1, OP_XSWAP = 2, OP_PHASE = 3, OP_ROT = 4 }; // OP_ROT: real rotation [[c,-s],[s,c]], m[0] = c, m[1] = s

template <typename R> struct alignas(16) DevOp {
    uint64_t omask, oval; // predicate on the tile's global base index (qubits outside the tile)
    // --- one 16-byte group, fetched with a single LDS.128 ---
    uint32_t code;    // opcode | CODE_HAS_SB
    uint32_t emask;   // single ops: bit e set = register amplitude e satisfies the register-resident controls
                      // OPC_STAGE: hmask | slotMask << 5 | anyMembers << 10
    uint32_t lmaskSb; // predicate on the sub-block base (tile-local amplitude bits outside the register set)
    uint32_t lvalSb;
    R m[8];           // inline, so that its loads do not wait for the header
};
struct DevPass {
    int opBegin, opEnd;
    int nsb;                       // number of sub-block index bits
    int nIt;                       // sub-blocks per thread
    unsigned char sbit[16];        // sub-block index bit i -> tile chunk bit
    unsigned short pswzB[MAX_NCH]; // register chunk e -> swizzled byte offset inside the tile
    unsigned short itoffC[16];     // iteration -> chunk-index contribution of the sub-block bits above the thread id
    unsigned int pad;
    uint64_t goff[MAX_NCH];        // register chunk e -> global amplitude offset (first / last pass move straight HBM <-> registers)
};

struct alignas(16) DevSweep {
    int nHigh;      // high qubits in the tile
    int lowAmpBits; // L: low qubits in the tile
    int kc;         // tile chunk bits actually used (<= KC)
    int nPass;
    int nOps;
    int hasScale;
    double scale;
    int nOuter;   // outer-only phases (DevOuterPhase records at outerOff)
    int outerOff;
    int reserved; // unused: kept because sizeof(DevSweep) counts against the program-size limit (how many ops fit a sweep)
    // scale: deferred scalar of the un-normalised Hadamard butterflies, applied once in the last pass
    int nSlots;   // per-tile phase table entries: slot 0 = tile scalar, slots 1.. = register-bit phases of the DIAG ops
    int scratchBytes; // shared memory behind the program: chunk-row offsets + the double-buffered phase table
    int directIn;  // 1: the first pass reads its sub-blocks straight from HBM; 0: coalesced copy into the smem tile first
    int directOut; // 1: the last pass writes straight to HBM; 0: through the smem tile
    int nMem;      // thread-level phase members (DevMember records at memOff)
    int memOff;
    int nRot;      // real rotations of the STAGE ops ((c, s) pairs at rotOff)
    int rotOff;
    int needFull;  // 1: the program holds XSWAP / general-matrix ops (launch the FULL kernel variant); 0: STAGE / phase ops only
    unsigned short slotBeg[MAX_SLOTS + 1]; // slot s multiplies the outer records [slotBeg[s], slotBeg[s+1])
    uint64_t highLow[MAX_HIGH]; // (2^q - 1) for push_apart of the tile base, ascending
    uint64_t highPow[MAX_HIGH]; // 2^q
    DevPass pass[MAX_PASS];
};

__device__ __forceinline__ uint4 ld_stream(const uint4* p)
{
    uint4 v;
    asm volatile("ld.global.cs.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ void st_stream(uint4* p, const uint4 v)
{
    asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// smem slot of tile chunk c: the 128-byte bank group (chunk bits 0..2) is XORed with every higher 3-bit field, so any
// three chunk bits from distinct classes {0,3,6,9}, {1,4,7,10}, {2,5,8,11} address eight different bank groups.  Linear over
// XOR: swz(a | b) = swz(a) ^ swz(b) for disjoint a, b (the passes combine a thread part and a register part that way).
__host__ __device__ __forceinline__ uint32_t swz(uint32_t c) { return c ^ ((c >> 3) & 7U) ^ ((c >> 6) & 7U) ^ ((c >> 9) & 7U); }

// ---------------------------------------------------------------------------------------------------------
// register representation of amplitudes.
//   fp32: one amplitude = one 64-bit register pair (re, im).  Hopper has no packed FP32 arithmetic, so f2add / f2mul /
//         f2fma apply the scalar FADD / FMUL / FFMA to each half (explicit _rn intrinsics: the compiler may not contract
//         or reorder them, so every lane rounds exactly as one packed .f32x2 lane would).  The pack/unpack movs are free:
//         the pair lives in two 32-bit registers either way.
//   fp64: plain double2 with DFMA.
// ---------------------------------------------------------------------------------------------------------
typedef unsigned long long ull;
__device__ __forceinline__ ull pk(float lo, float hi)
{
    ull r;
    asm("mov.b64 %0, {%1,%2};" : "=l"(r) : "f"(lo), "f"(hi));
    return r;
}
__device__ __forceinline__ ull swp64(ull v)
{
    float lo, hi;
    asm("mov.b64 {%0,%1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
    return pk(hi, lo);
}
__device__ __forceinline__ float2 upk(ull v)
{
    float2 f;
    asm("mov.b64 {%0,%1}, %2;" : "=f"(f.x), "=f"(f.y) : "l"(v));
    return f;
}
__device__ __forceinline__ ull f2add(ull a, ull b)
{
    const float2 x = upk(a), y = upk(b);
    return pk(__fadd_rn(x.x, y.x), __fadd_rn(x.y, y.y));
}
__device__ __forceinline__ ull f2mul(ull a, ull b)
{
    const float2 x = upk(a), y = upk(b);
    return pk(__fmul_rn(x.x, y.x), __fmul_rn(x.y, y.y));
}
__device__ __forceinline__ ull f2fma(ull a, ull b, ull c)
{
    const float2 x = upk(a), y = upk(b), z = upk(c);
    return pk(__fmaf_rn(x.x, y.x, z.x), __fmaf_rn(x.y, y.y, z.y));
}

template <typename R> struct AmpOps;
template <> struct AmpOps<float> {
    typedef ull A;
    typedef ulonglong2 Chunk; // 16 bytes = 2 amplitudes
    static constexpr int APC = 2;
    struct Ph {
        ull xx, ny; // (x, x), (-y, y)
    };
    static __device__ __forceinline__ Ph mkph(float x, float y) { return Ph{ pk(x, x), pk(-y, y) }; }
    static __device__ __forceinline__ A mulc(A a, const Ph& p) { return f2fma(a, p.xx, f2mul(swp64(a), p.ny)); }
    static __device__ __forceinline__ A macc(A a, const Ph& p, A acc) { return f2fma(a, p.xx, f2fma(swp64(a), p.ny, acc)); }
    static __device__ __forceinline__ void had(A& x, A& y)
    {
        x = f2add(x, y);
        y = f2fma(y, pk(-2.0f, -2.0f), x);
    }
    static __device__ __forceinline__ void rot(A& x, A& y, float c, float s)
    {
        const ull cc = pk(c, c), ss = pk(s, s), ns = pk(-s, -s);
        const A nx = f2fma(x, cc, f2mul(y, ns));
        y = f2fma(y, cc, f2mul(x, ss));
        x = nx;
    }
    static __device__ __forceinline__ A scale(A a, float s) { return f2mul(a, pk(s, s)); }
    static __device__ __forceinline__ A unit() { return pk(1.0f, 0.0f); }
    static __device__ __forceinline__ Ph toph(A a)
    {
        float x, y;
        asm("mov.b64 {%0,%1}, %2;" : "=f"(x), "=f"(y) : "l"(a));
        return mkph(x, y);
    }
    static __device__ __forceinline__ void get(const Chunk& c, A* a)
    {
        a[0] = c.x;
        a[1] = c.y;
    }
    static __device__ __forceinline__ Chunk put(const A* a)
    {
        Chunk c;
        c.x = a[0];
        c.y = a[1];
        return c;
    }
};
template <> struct AmpOps<double> {
    typedef double2 A;
    typedef double2 Chunk; // 16 bytes = 1 amplitude
    static constexpr int APC = 1;
    struct Ph {
        double x, y;
    };
    static __device__ __forceinline__ Ph mkph(double x, double y) { return Ph{ x, y }; }
    static __device__ __forceinline__ A mulc(A a, const Ph& p) { return make_double2(a.x * p.x - a.y * p.y, a.x * p.y + a.y * p.x); }
    static __device__ __forceinline__ A macc(A a, const Ph& p, A acc)
    {
        return make_double2(fma(a.x, p.x, fma(-a.y, p.y, acc.x)), fma(a.x, p.y, fma(a.y, p.x, acc.y)));
    }
    static __device__ __forceinline__ void had(A& x, A& y)
    {
        x.x += y.x;
        x.y += y.y;
        y.x = fma(y.x, -2.0, x.x);
        y.y = fma(y.y, -2.0, x.y);
    }
    static __device__ __forceinline__ void rot(A& x, A& y, double c, double s)
    {
        const A nx = make_double2(fma(c, x.x, -s * y.x), fma(c, x.y, -s * y.y));
        y = make_double2(fma(c, y.x, s * x.x), fma(c, y.y, s * x.y));
        x = nx;
    }
    static __device__ __forceinline__ A scale(A a, double s) { return make_double2(a.x * s, a.y * s); }
    static __device__ __forceinline__ A unit() { return make_double2(1.0, 0.0); }
    static __device__ __forceinline__ Ph toph(A a) { return Ph{ a.x, a.y }; }
    static __device__ __forceinline__ void get(const Chunk& c, A* a) { a[0] = c; }
    static __device__ __forceinline__ Chunk put(const A* a) { return a[0]; }
};

template <typename R> struct Apc {
    static constexpr int v = AmpOps<R>::APC;
};

// ---- in-register gate bodies: JR = register-bit index of the target ------------------------------------------------
template <typename R, int JR, int NA> __device__ __forceinline__ void app_had(typename AmpOps<R>::A (&a)[NA])
{
#pragma unroll
    for (int e = 0; e < NA; ++e) {
        if (!(e & (1 << JR))) {
            AmpOps<R>::had(a[e], a[e | (1 << JR)]);
        }
    }
}
// real rotation [[c, -s], [s, c]] on register bit JR: half the arithmetic of a general 2x2 per amplitude pair
template <typename R, int JR, int NA> __device__ __forceinline__ void app_rot(typename AmpOps<R>::A (&a)[NA], R c, R s)
{
    typedef AmpOps<R> O;
#pragma unroll
    for (int e = 0; e < NA; ++e) {
        if (!(e & (1 << JR))) {
            O::rot(a[e], a[e | (1 << JR)], c, s);
        }
    }
}
template <typename R, int JR, int NA, bool PRED>
__device__ __forceinline__ void app_general(typename AmpOps<R>::A (&a)[NA], const R* __restrict__ m, uint32_t em)
{
    typedef AmpOps<R> O;
    typedef typename O::A A;
    const typename O::Ph m0 = O::mkph(m[0], m[1]), m1 = O::mkph(m[2], m[3]), m2 = O::mkph(m[4], m[5]), m3 = O::mkph(m[6], m[7]);
#pragma unroll
    for (int e = 0; e < NA; ++e) {
        if (!(e & (1 << JR))) {
            const A x = a[e], y = a[e | (1 << JR)];
            const A nx = O::macc(y, m1, O::mulc(x, m0));
            const A ny = O::macc(y, m3, O::mulc(x, m2));
            if (PRED) {
                const bool p = (em >> e) & 1U;
                a[e] = p ? nx : x;
                a[e | (1 << JR)] = p ? ny : y;
            } else {
                a[e] = nx;
                a[e | (1 << JR)] = ny;
            }
        }
    }
}
template <typename R, int JR, int NA> __device__ __forceinline__ void app_xswap(typename AmpOps<R>::A (&a)[NA], uint32_t em)
{
    typedef typename AmpOps<R>::A A;
#pragma unroll
    for (int e = 0; e < NA; ++e) {
        if (!(e & (1 << JR))) {
            const bool p = (em >> e) & 1U;
            const A x = a[e], y = a[e | (1 << JR)];
            a[e] = p ? y : x;
            a[e | (1 << JR)] = p ? x : y;
        }
    }
}
template <typename R, int JR, int NA>
__device__ __forceinline__ void app_phase_reg(typename AmpOps<R>::A (&a)[NA], const typename AmpOps<R>::Ph& ph)
{
#pragma unroll
    for (int e = 0; e < NA; ++e) {
        if (e & (1 << JR)) {
            a[e] = AmpOps<R>::mulc(a[e], ph);
        }
    }
}

template <typename R, int JA, int JB, int NA>
__device__ __forceinline__ void app_phase_pair(typename AmpOps<R>::A (&a)[NA], const typename AmpOps<R>::Ph& ph)
{
#pragma unroll
    for (int e = 0; e < NA; ++e) {
        if ((e & (1 << JA)) && (e & (1 << JB))) {
            a[e] = AmpOps<R>::mulc(a[e], ph);
        }
    }
}

// thread-level phase member of a STAGE group
template <typename R> struct alignas(16) DevMember {
    uint64_t omask, oval; // outer predicate, evaluated once per tile (preamble) into the effective (mask, val) table
    uint32_t lmask, lval; // predicate on the sub-block base (thread bits)
    R ph[2];
};

template <typename R, int NA, int VAR>
__device__ __forceinline__ void exec_op(typename AmpOps<R>::A (&a)[NA], const DevOp<R>& op, const uint4 hd, uint32_t xsb,
    const R* __restrict__ tileScale, const DevMember<R>* __restrict__ members, const uint2* __restrict__ eff, const R* __restrict__ rotTab)
{
    typedef AmpOps<R> O;
    typedef typename O::A A;
    constexpr bool FULL = (VAR == 2);  // swap / general-matrix ops compiled in
    constexpr bool ROT = (VAR >= 1);   // stages may hold real rotations
    const R* m = op.m;
#define SV_J(J) (((1 << (J)) < NA) ? (J) : 0)
#define SV_CASES(J)                                                                                                    \
    case K_XSWAP * 5 + J:                                                                                              \
        app_xswap<R, SV_J(J), NA>(a, em);                                                                              \
        break;                                                                                                         \
    case K_GEN_U * 5 + J:                                                                                              \
        app_general<R, SV_J(J), NA, false>(a, m, em);                                                                  \
        break;                                                                                                         \
    case K_GEN_P * 5 + J:                                                                                              \
        app_general<R, SV_J(J), NA, true>(a, m, em);                                                                   \
        break;
#define SV_PAIR(K, J)                                                                                                  \
    case OPC_PH2 + (K) * ((K)-1) / 2 + (J):                                                                            \
        if (tp && ((1 << (K)) < NA)) {                                                                                 \
            app_phase_pair<R, SV_J(J), SV_J(K), NA>(a, O::mkph(m[0], m[1]));                                           \
        }                                                                                                              \
        break;
    if ((hd.x & 0xffU) == OPC_STAGE) {
        const uint32_t hm = hd.y & ST_MASK, sm = (hd.y >> ST_SM_SHIFT) & ST_MASK, act = (hd.y >> ST_ACT_SHIFT) & ST_MASK,
                       rm = ROT ? ((hd.y >> ST_RM_SHIFT) & ST_MASK) : 0U;
        uint32_t slot = hd.z, mk = hd.w & 0xffffU, ri = hd.w >> 16;
        if (!FULL && !(hd.y & (1U << ST_ANY_BIT))) {
            // the common shape: per-tile slot phases and butterflies only (no thread-level members)
#define SV_STAGE_FAST(J)                                                                                               \
    if (((1 << (J)) < NA) && ((act >> (J)) & 1U)) {                                                                    \
        if ((sm >> (J)) & 1U) {                                                                                        \
            const R px = tileScale[2U * slot], py = tileScale[2U * slot + 1U];                                         \
            ++slot;                                                                                                    \
            if (px != (R)1 || py != (R)0) {                                                                            \
                app_phase_reg<R, SV_J(J), NA>(a, O::mkph(px, py));                                                     \
            }                                                                                                          \
        }                                                                                                              \
        if ((hm >> (J)) & 1U) {                                                                                        \
            if (ROT && ((rm >> (J)) & 1U)) {                                                                           \
                app_rot<R, SV_J(J), NA>(a, rotTab[2U * ri], rotTab[2U * ri + 1U]);                                     \
                ++ri;                                                                                                  \
            } else {                                                                                                   \
                app_had<R, SV_J(J), NA>(a);                                                                            \
            }                                                                                                          \
        }                                                                                                              \
    }
            SV_STAGE_FAST(0)
            SV_STAGE_FAST(1)
            SV_STAGE_FAST(2)
            SV_STAGE_FAST(3)
            SV_STAGE_FAST(4)
            SV_STAGE_FAST(5)
#undef SV_STAGE_FAST
            return;
        }
        const uint32_t cnts = (hd.y & (1U << ST_ANY_BIT)) ? *reinterpret_cast<const uint32_t*>(op.m) : 0U;
        // product of the thread-level members [mk, mk + c) that fire for this thread, times (px, py)
#define SV_MEMBERS(c)                                                                                                  \
    _Pragma("unroll 1") for (uint32_t k = 0; k < (c); ++k, ++mk) {                                                                         \
        const uint2 e = eff[mk];                                                                                       \
        const R qx = members[mk].ph[0], qy = members[mk].ph[1];                                                        \
        if ((xsb & e.x) == e.y) {                                                                                      \
            const R nx = px * qx - py * qy;                                                                            \
            py = px * qy + py * qx;                                                                                    \
            px = nx;                                                                                                   \
        }                                                                                                              \
    }
        {
            const uint32_t c = cnts & ST_CNT_MASK;
            if (c) {
                R px = (R)1, py = (R)0;
                SV_MEMBERS(c)
                if (px != (R)1 || py != (R)0) {
                    const typename O::Ph ph = O::mkph(px, py);
#pragma unroll
                    for (int e = 0; e < NA; ++e) {
                        a[e] = O::mulc(a[e], ph);
                    }
                }
            }
        }
#define SV_STAGE_BIT(J)                                                                                                \
    if (((1 << (J)) < NA) && ((act >> (J)) & 1U)) {                                                                    \
        const uint32_t c = (cnts >> (ST_CNT_BITS * ((J) + 1))) & ST_CNT_MASK;                                          \
        if (((sm >> (J)) & 1U) | c) {                                                                                  \
            R px = (R)1, py = (R)0;                                                                                    \
            if ((sm >> (J)) & 1U) {                                                                                    \
                px = tileScale[2U * slot];                                                                             \
                py = tileScale[2U * slot + 1U];                                                                        \
                ++slot;                                                                                                \
            }                                                                                                          \
            SV_MEMBERS(c)                                                                                              \
            if (px != (R)1 || py != (R)0) {                                                                            \
                app_phase_reg<R, SV_J(J), NA>(a, O::mkph(px, py));                                                     \
            }                                                                                                          \
        }                                                                                                              \
        if ((hm >> (J)) & 1U) {                                                                                        \
            if (ROT && ((rm >> (J)) & 1U)) {                                                                           \
                app_rot<R, SV_J(J), NA>(a, rotTab[2U * ri], rotTab[2U * ri + 1U]);                                     \
                ++ri;                                                                                                  \
            } else {                                                                                                   \
                app_had<R, SV_J(J), NA>(a);                                                                            \
            }                                                                                                          \
        }                                                                                                              \
    }
        SV_STAGE_BIT(0)
        SV_STAGE_BIT(1)
        SV_STAGE_BIT(2)
        SV_STAGE_BIT(3)
        SV_STAGE_BIT(4)
        SV_STAGE_BIT(5)
#undef SV_STAGE_BIT
#undef SV_MEMBERS
        return;
    }
    bool tp = true;
    if (hd.x & CODE_HAS_SB) {
        tp = (xsb & hd.z) == hd.w;
    }
    // register-amplitude predicate mask
    const uint32_t em = tp ? hd.y : 0U;
    if (FULL && (hd.x & 0xffU) < OPC_PHGEN) {
        switch (hd.x & 0xffU) {
            SV_CASES(0)
            SV_CASES(1)
            SV_CASES(2)
            SV_CASES(3)
            SV_CASES(4)
        default:
            break;
        }
        return;
    }
    switch (hd.x & 0xffU) {
    case OPC_SCALE: {
        const typename O::Ph sc = O::mkph(tileScale[0], tileScale[1]);
#pragma unroll
        for (int e = 0; e < NA; ++e) {
            a[e] = O::mulc(a[e], sc);
        }
    } break;
        SV_PAIR(1, 0)
        SV_PAIR(2, 0)
        SV_PAIR(2, 1)
        SV_PAIR(3, 0)
        SV_PAIR(3, 1)
        SV_PAIR(3, 2)
        SV_PAIR(4, 0)
        SV_PAIR(4, 1)
        SV_PAIR(4, 2)
        SV_PAIR(4, 3)
        SV_PAIR(5, 0)
        SV_PAIR(5, 1)
        SV_PAIR(5, 2)
        SV_PAIR(5, 3)
        SV_PAIR(5, 4)
    case OPC_PHGEN: {
        const typename O::Ph ph = O::mkph(m[0], m[1]);
#pragma unroll
        for (int e = 0; e < NA; ++e) {
            const A v = O::mulc(a[e], ph);
            a[e] = ((em >> e) & 1U) ? v : a[e];
        }
    } break;
    default:
        break;
    }
#undef SV_PAIR
#undef SV_CASES
#undef SV_J
}

// outer-only diagonal gate (every qubit of its predicate lies outside the tile): uniform per tile, folded into one
// per-tile complex scalar that is applied together with the deferred Hadamard scale in the last pass
template <typename R> struct DevOuterPhase {
    uint64_t omask, oval;
    R ph[2];
    R pad[(sizeof(R) == 4) ? 2 : 2];
};

constexpr int MAX_OUTER = 192;

// Staged tile copies (used when the first / last pass has register bits on low chunk bits): coalesced HBM <-> swizzled
// smem.  Kept out of line so that their registers do not weigh on the pass loop.
// Source address of amplitude index i of this rank's NEW page while a pull re-page is pending (PullArgs): the victim bits of i
// name the rank whose old page holds it, at index i with the victim bits replaced by this rank's bits.
template <typename C> __device__ __forceinline__ const C* pull_src(const PullArgs& pa, uint64_t i)
{
    unsigned r = (unsigned)((i >> pa.vb[0]) & 1ULL);
    if (pa.k > 1) {
        r |= (unsigned)((i >> pa.vb[1]) & 1ULL) << 1;
    }
    if (pa.k > 2) {
        r |= (unsigned)((i >> pa.vb[2]) & 1ULL) << 2;
    }
    return reinterpret_cast<const C*>(pa.peers[r]) + ((i & ~pa.vmask) | pa.rankDep);
}

template <typename R>
__device__ __noinline__ void stage_in_pull(const PullArgs& pa, uint64_t base, unsigned char* tileB, const uint64_t* rowOff,
    uint32_t nChunk, int lcb, uint32_t colMask, int tid)
{
    typedef typename Cx<R>::type C;
    constexpr int APC = AmpOps<R>::APC;
    constexpr int NT = FUSED_NT;
    for (uint32_t c0 = (uint32_t)tid; c0 < nChunk; c0 += 4U * NT) {
        uint4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const uint32_t c = c0 + (uint32_t)u * NT;
            if (c < nChunk) {
                v[u] = ld_stream(reinterpret_cast<const uint4*>(pull_src<C>(pa, base + rowOff[c >> lcb] + (uint64_t)(c & colMask) * APC)));
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const uint32_t c = c0 + (uint32_t)u * NT;
            if (c < nChunk) {
                *reinterpret_cast<uint4*>(tileB + ((size_t)swz(c) << 4)) = v[u];
            }
        }
    }
}

template <typename R>
__device__ __noinline__ void stage_in(const typename Cx<R>::type* __restrict__ tilePsi, unsigned char* tileB, const uint64_t* rowOff,
    uint32_t nChunk, int lcb, uint32_t colMask, int tid)
{
    constexpr int APC = AmpOps<R>::APC;
    constexpr int NT = FUSED_NT;
    if (nChunk >= 8U * NT) {
        for (uint32_t c0 = (uint32_t)tid; c0 < nChunk; c0 += 8U * NT) {
            uint4 v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const uint32_t c = c0 + (uint32_t)u * NT;
                v[u] = ld_stream(reinterpret_cast<const uint4*>(tilePsi + rowOff[c >> lcb] + (uint64_t)(c & colMask) * APC));
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const uint32_t c = c0 + (uint32_t)u * NT;
                *reinterpret_cast<uint4*>(tileB + ((size_t)swz(c) << 4)) = v[u];
            }
        }
    } else {
        for (uint32_t c = (uint32_t)tid; c < nChunk; c += NT) {
            *reinterpret_cast<uint4*>(tileB + ((size_t)swz(c) << 4)) =
                ld_stream(reinterpret_cast<const uint4*>(tilePsi + rowOff[c >> lcb] + (uint64_t)(c & colMask) * APC));
        }
    }
}
template <typename R>
__device__ __noinline__ void stage_out(typename Cx<R>::type* __restrict__ tilePsi, const unsigned char* tileB, const uint64_t* rowOff,
    uint32_t nChunk, int lcb, uint32_t colMask, int tid)
{
    constexpr int APC = AmpOps<R>::APC;
    constexpr int NT = FUSED_NT;
#pragma unroll 4
    for (uint32_t c = (uint32_t)tid; c < nChunk; c += NT) {
        st_stream(reinterpret_cast<uint4*>(tilePsi + rowOff[c >> lcb] + (uint64_t)(c & colMask) * APC),
            *reinterpret_cast<const uint4*>(tileB + ((size_t)swz(c) << 4)));
    }
}

// PULL: the sweep also performs a pending re-page (PullArgs): its first pass (or the staged tile copy) reads every chunk through
// the peer mapping that holds it, its last pass writes this rank's other page; everything between is unchanged.
template <typename R, int VAR, bool PULL = false>
__global__ void __launch_bounds__(FUSED_NT, FUSED_MINB)
    k_fused_sweep(typename Cx<R>::type* __restrict__ psi, const unsigned char* __restrict__ prog, uint32_t progBytes, uint64_t nTiles,
        const __grid_constant__ PullArgs pull)
{
    typedef typename Cx<R>::type C;
    typedef AmpOps<R> O;
    typedef typename O::A A;
    typedef typename O::Chunk Chunk;
    constexpr int APC = O::APC;
    constexpr int NT = FUSED_NT;
    constexpr int NCH = 1 << FUSED_RB;
    constexpr int NA = NCH * APC;
    static_assert(NA <= MAX_NA && NCH <= MAX_NCH, "register sub-block too large");
    static_assert(NT > 128, "the per-tile preamble uses warps 0..3 for the ballots and the tile scalar, the rest for the table slots");
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char* tileB = smem;
    unsigned char* sprog = smem + ((size_t)16 << FUSED_KC);
    __shared__ uint32_t ballots[2][4]; // double-buffered by tile parity (like tileTab) so that one barrier per tile is enough

    const int tid = threadIdx.x;
    for (uint32_t i = tid; i < progBytes / 16; i += NT) {
        reinterpret_cast<uint4*>(sprog)[i] = reinterpret_cast<const uint4*>(prog)[i];
    }
    __syncthreads();
    const DevSweep& sw = *reinterpret_cast<const DevSweep*>(sprog);
    const DevOp<R>* ops = reinterpret_cast<const DevOp<R>*>(sprog + sizeof(DevSweep));
    const int kc = sw.kc;
    const uint32_t nChunk = 1U << kc;
    const int lcb = sw.lowAmpBits - (APC == 2 ? 1 : 0); // low (contiguous) chunk bits
    const uint32_t colMask = (1U << lcb) - 1U;
    // scratch behind the program: global amplitude offset of each chunk row of the tile (depends only on the sweep's high
    // qubits), then the per-tile phase table ([0..1] tile scalar, then the DIAG register-bit phases), double-buffered
    const uint32_t nRows = nChunk >> lcb;
    uint64_t* const rowOff = reinterpret_cast<uint64_t*>(sprog + progBytes);
    R* const tileTab = reinterpret_cast<R*>(rowOff + nRows);
    const uint32_t tabStride = 2U * (uint32_t)sw.nSlots;
    for (uint32_t r = tid; r < nRows; r += NT) {
        uint64_t off = 0;
        for (int h = 0; h < sw.nHigh; ++h) {
            if ((r >> h) & 1U) {
                off |= sw.highPow[h];
            }
        }
        rowOff[r] = off;
    }
    const uint32_t nSub = nChunk >> FUSED_RB;
    const int nOps = sw.nOps;
    const int nOuter = sw.nOuter;
    const int nPass = sw.nPass;
    const DevOuterPhase<R>* outer = reinterpret_cast<const DevOuterPhase<R>*>(sprog + sw.outerOff);
    // thread-level phase members of the STAGE ops: static records in the program, per-tile effective (mask, val) pairs
    // (double-buffered by tile parity like the phase table) behind it
    const int nMem = sw.nMem;
    const DevMember<R>* members = reinterpret_cast<const DevMember<R>*>(sprog + sw.memOff);
    uint2* const effTab = reinterpret_cast<uint2*>(tileTab + 2U * tabStride);
    const R* const rotTab = reinterpret_cast<const R*>(sprog + sw.rotOff); // (c, s) of the stages' real rotations
    // tile-chunk index of this thread's sub-block base in every pass (depends on the pass's bit assignment only, not on the tile)
    unsigned short* const depTab = reinterpret_cast<unsigned short*>(effTab + 2U * (uint32_t)nMem);
    for (int p = 0; p < nPass; ++p) {
        const DevPass& ps = sw.pass[p];
        const int nb = ps.nsb < 8 ? ps.nsb : 8;
        uint32_t dep = 0;
        for (int i = 0; i < nb; ++i) {
            dep |= ((tid >> i) & 1U) << ps.sbit[i];
        }
        depTab[p * NT + tid] = (unsigned short)dep;
    }
    __syncthreads();

    // tile t = blockIdx.x + k * gridDim.x; only the 32-bit k is carried across tiles (a CTA never sees 2^32 64 KB tiles of a state
    // that fits in device memory), which keeps one more register free for the pass loop
    for (uint32_t k = 0;; ++k) {
        const uint64_t t = blockIdx.x + (uint64_t)k * gridDim.x;
        if (t >= nTiles) {
            break;
        }
        const uint32_t par = k & 1U;
        uint64_t base = t << sw.lowAmpBits;
        for (int h = 0; h < sw.nHigh; ++h) {
            const uint64_t lo = base & sw.highLow[h];
            base = ((base ^ lo) << 1) | lo;
        }
        C* const tilePsi = (PULL ? reinterpret_cast<C*>(pull.out) : psi) + base; // PULL: the tile's place in the OUT page
        R* const tileScale = tileTab + par * tabStride;
        // ---- per-tile preamble ------------------------------------------------------------------------------------
        // warps 0..2: which ops act on this tile (predicates on qubits outside the tile are uniform per tile)
        // warp 3   : product of the outer-only phases that fire for this tile, times the deferred Hadamard scale
        // warps 4..: one thread per DIAG table slot
        if (tid < 96) {
            const DevOp<R>& aop = ops[tid < nOps ? tid : 0];
            const bool act = (tid < nOps) && ((base & aop.omask) == aop.oval);
            const uint32_t bal = __ballot_sync(0xffffffffU, act);
            if ((tid & 31) == 0) {
                ballots[par][tid >> 5] = bal;
            }
        } else if (tid < 128) {
            R fx = (R)1, fy = (R)0;
            for (int i = tid - 96; i < nOuter; i += 32) {
                const DevOuterPhase<R>& op = outer[i];
                if ((base & op.omask) == op.oval) {
                    const R nx = fx * op.ph[0] - fy * op.ph[1];
                    fy = fx * op.ph[1] + fy * op.ph[0];
                    fx = nx;
                }
            }
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) {
                const R ox = __shfl_xor_sync(0xffffffffU, fx, d), oy = __shfl_xor_sync(0xffffffffU, fy, d);
                const R nx = fx * ox - fy * oy;
                fy = fx * oy + fy * ox;
                fx = nx;
            }
            if (tid == 96) {
                tileScale[0] = fx * (R)sw.scale;
                tileScale[1] = fy * (R)sw.scale;
            }
        }
        // table slots 1..: product (in double) of the member phases that fire for this tile; one thread per slot, the threads
        // beyond the four role warps first
        for (int sl = 1 + (tid >= 128 ? tid - 128 : tid + NT - 128); sl < sw.nSlots; sl += NT) {
            double fx = 1.0, fy = 0.0;
            for (int i = sw.slotBeg[sl], e = sw.slotBeg[sl + 1]; i < e; ++i) {
                const DevOuterPhase<R>& op = outer[i];
                if ((base & op.omask) == op.oval) {
                    const double nx = fx * (double)op.ph[0] - fy * (double)op.ph[1];
                    fy = fx * (double)op.ph[1] + fy * (double)op.ph[0];
                    fx = nx;
                }
            }
            tileScale[2 * sl] = (R)fx;
            tileScale[2 * sl + 1] = (R)fy;
        }
        {
            // members whose outer predicate fails on this tile can never match: (mask 0, val 1)
            uint2* const eff = effTab + par * (uint32_t)nMem;
            for (int i = tid; i < nMem; i += NT) {
                const DevMember<R>& mb = members[i];
                const bool ok = (base & mb.omask) == mb.oval;
                eff[i] = ok ? make_uint2(mb.lmask, mb.lval) : make_uint2(0U, 1U);
            }
        }
        if (!sw.directIn) {
            // staged input (register bits of the first pass sit on low chunk bits, where per-thread HBM access would
            // split sectors): coalesced copy global -> swizzled smem.  The extra barrier keeps slow warps of the
            // previous tile from still reading the tile area.
            __syncthreads();
            if (PULL) {
                stage_in_pull<R>(pull, base, tileB, rowOff, nChunk, lcb, colMask, tid);
            } else {
                stage_in<R>(tilePsi, tileB, rowOff, nChunk, lcb, colMask, tid);
            }
        }
        // The barrier publishes the tables (and the staged tile) and closes the previous tile: nobody still reads the
        // tile area of smem.
        __syncthreads();
        // ---- passes: the first one reads its sub-blocks straight from HBM, the last one writes straight back; only the
        // hand-over between passes goes through the (swizzled) tile in shared memory --------------------------------------
        for (int p = 0; p < nPass; ++p) {
            const DevPass& ps = sw.pass[p];
            const bool fromGlobal = (p == 0) && sw.directIn, toGlobal = (p == nPass - 1) && sw.directOut;
            const uint32_t dep = depTab[p * NT + tid];
            const int opBegin = ps.opBegin, opEnd = ps.opEnd;
            const uint2* const effCur = effTab + par * (uint32_t)nMem;
            for (int it = 0; it < ps.nIt; ++it) {
                if ((uint32_t)(it * NT + tid) >= nSub) {
                    break;
                }
                const uint32_t sbc = dep | ps.itoffC[it];
                const uint32_t swb = swz(sbc) << 4;
                C* const gsub = tilePsi + rowOff[sbc >> lcb] + (uint64_t)(sbc & colMask) * APC;
                A a[NA];
                if (fromGlobal && PULL) {
                    const uint64_t gi = base + rowOff[sbc >> lcb] + (uint64_t)(sbc & colMask) * APC;
#pragma unroll
                    for (int e = 0; e < NCH; ++e) {
                        const uint4 v = ld_stream(reinterpret_cast<const uint4*>(pull_src<C>(pull, gi + ps.goff[e])));
                        O::get(*reinterpret_cast<const Chunk*>(&v), &a[e * APC]);
                    }
                } else if (fromGlobal) {
#pragma unroll
                    for (int e = 0; e < NCH; ++e) {
                        const uint4 v = ld_stream(reinterpret_cast<const uint4*>(gsub + ps.goff[e]));
                        O::get(*reinterpret_cast<const Chunk*>(&v), &a[e * APC]);
                    }
                } else {
#pragma unroll
                    for (int e = 0; e < NCH; ++e) {
                        const Chunk c = *reinterpret_cast<const Chunk*>(tileB + (swb ^ ps.pswzB[e]));
                        O::get(c, &a[e * APC]);
                    }
                }
                const uint32_t xsb = sbc * APC;
                // linear walk over the pass's ops; only ops with a predicate on outer qubits look at the per-tile ballot
#pragma unroll 1
                for (int o = opBegin; o < opEnd; ++o) {
                    const uint4 hd = *reinterpret_cast<const uint4*>(&ops[o].code);
                    if ((hd.x & CODE_HAS_OUTER) && !((ballots[par][o >> 5] >> (o & 31)) & 1U)) {
                        continue;
                    }
                    exec_op<R, NA, VAR>(a, ops[o], hd, xsb, tileScale, members, effCur, rotTab);
                }
                if (toGlobal) {
#pragma unroll
                    for (int e = 0; e < NCH; ++e) {
                        const Chunk c = O::put(&a[e * APC]);
                        st_stream(reinterpret_cast<uint4*>(gsub + ps.goff[e]), *reinterpret_cast<const uint4*>(&c));
                    }
                } else {
#pragma unroll
                    for (int e = 0; e < NCH; ++e) {
                        *reinterpret_cast<Chunk*>(tileB + (swb ^ ps.pswzB[e])) = O::put(&a[e * APC]);
                    }
                }
            }
            if (!toGlobal) {
                __syncthreads();
            }
        }
        if (!sw.directOut) {
            // staged output: swizzled smem -> global, coalesced (the barrier above closed the last pass)
            stage_out<R>(tilePsi, tileB, rowOff, nChunk, lcb, colMask, tid);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// host-side scheduler
// ---------------------------------------------------------------------------------------------------------
struct HostOp {
    int kind;       // OP_*
    int tq;         // target qubit (-1 for OP_PHASE)
    uint64_t cmask; // predicate mask over qubits (controls; for OP_PHASE includes the phased qubit)
    uint64_t cval;
    double m[8];
};

static inline uint64_t bitq(int q) { return 1ULL << q; }

static uint64_t rewrite_ops(std::vector<HostOp>& ops);
// returns the mask of a trailing XMask that is better served by the dedicated sweep (launch_xmask) after the fused sweeps
static uint64_t lower_queue(const std::vector<GateOp>& q, std::vector<HostOp>& out)
{
    out.clear();
    out.reserve(q.size() * 2);
    for (const GateOp& g : q) {
        HostOp h;
        memset(&h, 0, sizeof(h));
        if (g.kind == 1) { // diagonal: one predicated phase per non-unit diagonal entry
            const bool one0 = (g.m[0] == 1.0 && g.m[1] == 0.0), one3 = (g.m[6] == 1.0 && g.m[7] == 0.0);
            const double n0 = g.m[0] * g.m[0] + g.m[1] * g.m[1];
            if (!one0 && n0 > 0.0) {
                // diag(d0, d3) under controls C  =  [C -> d0] . [C and target=1 -> d3 / d0]: every register-bit predicate the
                // kernel sees then asks for value 1 (a stage member), and the first factor has one qubit less
                h.kind = OP_PHASE;
                h.tq = -1;
                h.cmask = g.cmask;
                h.cval = g.cval;
                h.m[0] = g.m[0];
                h.m[1] = g.m[1];
                out.push_back(h);
                const double qx = (g.m[6] * g.m[0] + g.m[7] * g.m[1]) / n0, qy = (g.m[7] * g.m[0] - g.m[6] * g.m[1]) / n0;
                if (qx != 1.0 || qy != 0.0) {
                    h.cmask = g.cmask | bitq(g.target);
                    h.cval = g.cval | bitq(g.target);
                    h.m[0] = qx;
                    h.m[1] = qy;
                    out.push_back(h);
                }
                continue;
            }
            // d0 = 1 (or |d0| = 0): one predicated phase per remaining non-unit entry
            if (!one0) {
                h.kind = OP_PHASE;
                h.tq = -1;
                h.cmask = g.cmask | bitq(g.target);
                h.cval = g.cval;
                h.m[0] = g.m[0];
                h.m[1] = g.m[1];
                out.push_back(h);
            }
            if (!one3) {
                h.kind = OP_PHASE;
                h.tq = -1;
                h.cmask = g.cmask | bitq(g.target);
                h.cval = g.cval | bitq(g.target);
                h.m[0] = g.m[6];
                h.m[1] = g.m[7];
                out.push_back(h);
            }
            continue;
        }
        h.tq = g.target;
        h.cmask = g.cmask;
        h.cval = g.cval;
        memcpy(h.m, g.m, sizeof(h.m));
        const bool allReal = (g.m[1] == 0.0 && g.m[3] == 0.0 && g.m[5] == 0.0 && g.m[7] == 0.0);
        if (g.kind == 2 && g.m[2] == 1.0 && g.m[3] == 0.0 && g.m[4] == 1.0 && g.m[5] == 0.0) {
            h.kind = OP_XSWAP;
        } else if (!g.cmask && allReal && g.m[0] > 0.0 && g.m[0] == g.m[2] && g.m[0] == g.m[4] && g.m[6] == -g.m[0]) {
            h.kind = OP_HAD; // c * [[1,1],[1,-1]]: butterfly now, the scalar c is applied once per sweep
        } else {
            h.kind = OP_GENERAL;
        }
        out.push_back(h);
    }
    const uint64_t xtail = rewrite_ops(out);
    if (getenv("B200SV_FUSED_DEBUG")) {
        int cnt[5] = { 0, 0, 0, 0, 0 };
        for (const HostOp& h : out) {
            cnt[h.kind]++;
        }
        fprintf(stderr, "lowered: %zu gates -> %zu ops (general %d, hadamard %d, xswap %d, phase %d, rotation %d)\n", q.size(), out.size(), cnt[0],
            cnt[1], cnt[2], cnt[3], cnt[4]);
        if (atoi(getenv("B200SV_FUSED_DEBUG")) >= 2) {
            for (const HostOp& h : out) {
                fprintf(stderr, "   %s t=%d cmask=%llx cval=%llx m0=(%.3f,%.3f)\n", h.kind == OP_PHASE ? "PH" : (h.kind == OP_HAD ? "H " : (h.kind == OP_XSWAP ? "X " : (h.kind == OP_ROT ? "R " : "G "))),
                    h.tq, (unsigned long long)h.cmask, (unsigned long long)h.cval, h.m[0], h.m[1]);
            }
        }
    }
    return xtail;
}

// ---------------------------------------------------------------------------------------------------------
// Peephole rewrite of the lowered gate list (r2).  The sweep kernel is issue-bound, not HBM-bound, once a window holds
// more than a few gates, and the dearest op by far is the conditional register swap of an X-type gate (CNOT: 64 SEL +
// 32 MOV per 32-amplitude sub-block, and its target has to be a tile qubit).  Diagonal gates are index-only: they ride in
// any pass on any qubit and are free when their qubits lie outside the tile.  So the list is rewritten to an equivalent one
// with as few non-diagonal ops as possible:
//   R1  X-type (any controls) on target b   ->  H_b . Z-type(controls + b) . H_b      (H X H = Z)
//   R2  adjacent uncontrolled non-diagonal 1-qubit gates on the same qubit are multiplied (H.H = scalar, H.U / U.H / U.U' = one
//       general gate), so the Hadamards of R1 cancel against, or are absorbed by, the neighbouring single-qubit gates
//   R3  a general 1-qubit gate absorbs adjacent single-qubit phases on its qubit; equal-predicate phases are multiplied
// "Adjacent" = no op in between touches the qubit at all (so the two ops may be brought together without reordering
// anything that does not commute).  Products are taken in double.  The product of the whole list is unchanged.
// BASELINE's H/T/CNOT circuit turns into Hadamards + T/CZ phases only; quantum-volume layers into one general gate per
// qubit and layer + CZ phases.
// ---------------------------------------------------------------------------------------------------------
struct M22 {
    double m[8];
};
static inline M22 m22_mul(const double* a, const double* b) // a . b  (b acts first)
{
    M22 r;
    for (int i = 0; i < 2; ++i) {
        for (int j = 0; j < 2; ++j) {
            double re = 0, im = 0;
            for (int k = 0; k < 2; ++k) {
                const double ax = a[2 * (2 * i + k)], ay = a[2 * (2 * i + k) + 1];
                const double bx = b[2 * (2 * k + j)], by = b[2 * (2 * k + j) + 1];
                re += ax * bx - ay * by;
                im += ax * by + ay * bx;
            }
            r.m[2 * (2 * i + j)] = re;
            r.m[2 * (2 * i + j) + 1] = im;
        }
    }
    return r;
}
static inline bool is_had_form(const double* m)
{
    return m[1] == 0.0 && m[3] == 0.0 && m[5] == 0.0 && m[7] == 0.0 && m[0] > 0.0 && m[0] == m[2] && m[0] == m[4] && m[6] == -m[0];
}

static uint64_t rewrite_ops(std::vector<HostOp>& ops)
{
    std::vector<HostOp> out;
    std::vector<char> alive;
    out.reserve(ops.size() * 3);
    alive.reserve(ops.size() * 3);
    std::vector<int> hist[64]; // per qubit: indices (into out) of the live ops that touch it, ascending
    double gx = 1.0, gy = 0.0;  // global scalar (commutes with everything), emitted once at the end
    auto touches = [](const HostOp& h) { return h.cmask | (h.tq >= 0 ? bitq(h.tq) : 0ULL); };
    auto push = [&](const HostOp& h) {
        const int idx = (int)out.size();
        out.push_back(h);
        alive.push_back(1);
        for (uint64_t m = touches(h); m; m &= m - 1U) {
            hist[__builtin_ctzll(m)].push_back(idx);
        }
    };
    auto kill_last_on = [&](int b) { // the last live op touching b touches only b
        alive[(size_t)hist[b].back()] = 0;
        hist[b].pop_back();
    };
    auto is_u1 = [](const HostOp& h) { return (h.kind == OP_HAD || h.kind == OP_GENERAL || h.kind == OP_XSWAP) && !h.cmask; };
    auto emit_phase1 = [&](int b, int val, double px, double py) {
        if (px == 1.0 && py == 0.0) {
            return;
        }
        const double pn = px * px + py * py;
        if (val == 0 && pn > 0.0 && (hist[b].empty() || out[(size_t)hist[b].back()].kind != OP_GENERAL || out[(size_t)hist[b].back()].tq != b)) {
            // phase on (b = 0)  =  global scalar p  x  phase 1/p on (b = 1): the kernel's register-bit predicates ask for value 1
            const double nx = gx * px - gy * py;
            gy = gx * py + gy * px;
            gx = nx;
            val = 1;
            const double ix = px / pn, iy = -py / pn;
            px = ix;
            py = iy;
        }
        if (!hist[b].empty()) {
            HostOp& p = out[(size_t)hist[b].back()];
            if (p.kind == OP_GENERAL && !p.cmask && p.tq == b) { // R3: row scaling of the general gate
                for (int c = 0; c < 2; ++c) {
                    double* e = &p.m[2 * (2 * val + c)];
                    const double nx = e[0] * px - e[1] * py;
                    e[1] = e[0] * py + e[1] * px;
                    e[0] = nx;
                }
                return;
            }
            if (p.kind == OP_PHASE && p.cmask == bitq(b) && p.cval == (val ? bitq(b) : 0ULL)) {
                const double nx = p.m[0] * px - p.m[1] * py;
                p.m[1] = p.m[0] * py + p.m[1] * px;
                p.m[0] = nx;
                return;
            }
        }
        HostOp h;
        memset(&h, 0, sizeof(h));
        h.kind = OP_PHASE;
        h.tq = -1;
        h.cmask = bitq(b);
        h.cval = val ? bitq(b) : 0ULL;
        h.m[0] = px;
        h.m[1] = py;
        push(h);
    };
    // emit an uncontrolled 1-qubit matrix on b, merging with what is already there
    auto emit_u1 = [&](int b, const double* min) {
        M22 cur;
        memcpy(cur.m, min, sizeof(cur.m));
        auto is_x_form = [](const double* m) {
            return m[0] == 0 && m[1] == 0 && m[6] == 0 && m[7] == 0 && m[2] == 1.0 && m[3] == 0 && m[4] == 1.0 && m[5] == 0;
        };
        bool general = !is_had_form(cur.m) && !is_x_form(cur.m);
        for (;;) {
            if (hist[b].empty()) {
                break;
            }
            const HostOp& p = out[(size_t)hist[b].back()];
            if (is_u1(p) && p.tq == b) { // R2
                if (p.kind == OP_XSWAP && is_had_form(cur.m) && !general) {
                    // X then H  =  H then Z: keep the butterfly cheap instead of multiplying into a general gate
                    out[(size_t)hist[b].back()].kind = OP_HAD;
                    memcpy(out[(size_t)hist[b].back()].m, cur.m, sizeof(cur.m));
                    emit_phase1(b, 1, -1.0, 0.0);
                    return;
                }
                cur = m22_mul(cur.m, p.m);
                kill_last_on(b);
                general = !is_had_form(cur.m) && !is_x_form(cur.m);
                continue;
            }
            if (general && p.kind == OP_PHASE && p.cmask == bitq(b)) { // R3: column scaling
                const int val = p.cval ? 1 : 0;
                for (int r = 0; r < 2; ++r) {
                    double* e = &cur.m[2 * (2 * r + val)];
                    const double nx = e[0] * p.m[0] - e[1] * p.m[1];
                    e[1] = e[0] * p.m[1] + e[1] * p.m[0];
                    e[0] = nx;
                }
                kill_last_on(b);
                continue;
            }
            break;
        }
        const double* m = cur.m;
        const bool z1 = m[2] == 0 && m[3] == 0, z2 = m[4] == 0 && m[5] == 0;
        if (z1 && z2) { // diagonal
            if (m[0] == m[6] && m[1] == m[7]) {
                const double nx = gx * m[0] - gy * m[1];
                gy = gx * m[1] + gy * m[0];
                gx = nx;
            } else {
                emit_phase1(b, 0, m[0], m[1]);
                emit_phase1(b, 1, m[6], m[7]);
            }
            return;
        }
        HostOp h;
        memset(&h, 0, sizeof(h));
        h.tq = b;
        memcpy(h.m, m, sizeof(h.m));
        const bool z0 = m[0] == 0 && m[1] == 0, z3 = m[6] == 0 && m[7] == 0;
        if (is_had_form(m)) {
            h.kind = OP_HAD;
        } else if (z0 && z3 && m[2] == 1.0 && m[3] == 0.0 && m[4] == 1.0 && m[5] == 0.0) {
            h.kind = OP_XSWAP; // a product that happens to be X: left as a swap (no second rewrite)
        } else {
            h.kind = OP_GENERAL;
        }
        push(h);
    };
    static const double HS = 0.70710678118654752440;
    static const double HM[8] = { HS, 0, HS, 0, HS, 0, -HS, 0 };
    static const double XM[8] = { 0, 0, 1, 0, 1, 0, 0, 0 };
    // R4: a bare X travels forward through everything that uses its qubit only as a control / phase predicate (the predicate's
    // polarity flips), and two of them cancel.  QInterface::MACWrapper (include/qinterface.hpp:179-189) wraps every anti-controlled
    // gate in XMask ... XMask: here that costs nothing instead of two sweeps.
    uint64_t xpend = 0;
    auto emit_bare_x = [&](int q) {
        if (hist[q].empty() || out[(size_t)hist[q].back()].kind != OP_HAD || out[(size_t)hist[q].back()].tq != q) {
            emit_u1(q, XM); // next to a general gate (or to nothing): multiply / leave as a swap
        } else { // H X = Z-conjugate: H . (H Z H) -> Z H
            emit_u1(q, HM);
            emit_phase1(q, 1, -1.0, 0.0);
            emit_u1(q, HM);
        }
    };
    for (const HostOp& op0 : ops) {
        HostOp op = op0;
        op.cval ^= (op.cmask & xpend);
        if (op.kind == OP_XSWAP && !op.cmask) {
            xpend ^= bitq(op.tq);
            continue;
        }
        if (op.tq >= 0 && (xpend & bitq(op.tq))) {
            xpend &= ~bitq(op.tq);
            if (is_u1(op) && op.kind == OP_HAD) {
                emit_u1(op.tq, op.m); // X then H  =  H then Z
                emit_phase1(op.tq, 1, -1.0, 0.0);
                continue;
            }
            if (is_u1(op)) { // M . X: columns swapped
                double mx[8] = { op.m[2], op.m[3], op.m[0], op.m[1], op.m[6], op.m[7], op.m[4], op.m[5] };
                emit_u1(op.tq, mx);
                continue;
            }
            emit_bare_x(op.tq); // a controlled op on that target: the X has to be applied first
        }
        if (op.kind == OP_XSWAP) { // R1 (controlled X)
            emit_u1(op.tq, HM);
            HostOp z;
            memset(&z, 0, sizeof(z));
            z.kind = OP_PHASE;
            z.tq = -1;
            z.cmask = op.cmask | bitq(op.tq);
            z.cval = op.cval | bitq(op.tq);
            z.m[0] = -1.0;
            push(z);
            emit_u1(op.tq, HM);
        } else if (is_u1(op)) {
            emit_u1(op.tq, op.m);
        } else if (op.kind == OP_PHASE && op.cmask && !(op.cmask & (op.cmask - 1U))) {
            emit_phase1(__builtin_ctzll(op.cmask), op.cval ? 1 : 0, op.m[0], op.m[1]);
        } else if (op.kind == OP_PHASE && !op.cmask) {
            const double nx = gx * op.m[0] - gy * op.m[1];
            gy = gx * op.m[1] + gy * op.m[0];
            gx = nx;
        } else {
            push(op);
        }
    }
    uint64_t xtail = 0;
    if (__builtin_popcountll(xpend) > 4) {
        xtail = xpend; // a wide XMask that nothing absorbed: one dedicated permutation sweep beats that many fused swaps
    } else {
        for (uint64_t m = xpend; m; m &= m - 1U) {
            emit_bare_x(__builtin_ctzll(m));
        }
    }
    // R5: an uncontrolled UNITARY general gate is  g . diag(1, p_post) . [[c, -s], [s, c]] . diag(1, p_pre)  with real c, s >= 0.
    // The real rotation costs half the arithmetic of a general 2x2 per amplitude pair, runs inside a STAGE
    // (no dispatch of its own), and the two phases are ordinary diagonal ops: they merge with the CZ / T phases around them
    // and are applied lazily.  Quantum-volume layers (AI gates + CNOTs) become rotations + phases only: the flush is "light".
    std::vector<HostOp> res;
    res.reserve(out.size() + 1);
    for (size_t i = 0; i < out.size(); ++i) {
        if (!alive[i]) {
            continue;
        }
        const HostOp& h = out[i];
        if (h.kind == OP_GENERAL && !h.cmask) {
            const double* m = h.m;
            const double n00 = m[0] * m[0] + m[1] * m[1], n10 = m[4] * m[4] + m[5] * m[5];
            const double n01 = m[2] * m[2] + m[3] * m[3], n11 = m[6] * m[6] + m[7] * m[7];
            // unitary within rounding of the (possibly float-rounded) entries: unit columns, orthogonal
            const double ox = m[0] * m[2] + m[1] * m[3] + m[4] * m[6] + m[5] * m[7], oy = m[0] * m[3] - m[1] * m[2] + m[4] * m[7] - m[5] * m[6];
            if (fabs(n00 + n10 - 1.0) < 1e-5 && fabs(n01 + n11 - 1.0) < 1e-5 && fabs(ox) < 1e-5 && fabs(oy) < 1e-5 && n10 > 1e-24 && n01 > 1e-24) {
                const double c = sqrt(n00), sn = sqrt(n10);
                double g0x = 1.0, g0y = 0.0; // g = u00 / |u00| (1 when u00 = 0)
                if (c > 1e-12) {
                    g0x = m[0] / c;
                    g0y = m[1] / c;
                }
                // p_post = (u10 / g) / s,  p_pre = -(u01 / g) / s'   (s' = |u01|, equal to s for a unitary)
                const double s01 = sqrt(n01);
                const double ax = (m[4] * g0x + m[5] * g0y) / sn, ay = (m[5] * g0x - m[4] * g0y) / sn;
                const double bx = -(m[2] * g0x + m[3] * g0y) / s01, by = -(m[3] * g0x - m[2] * g0y) / s01;
                // fold |u01| != |u10| (rounding) into the rotation's sine: use their mean
                const double sm = 0.5 * (sn + s01);
                const double nx = gx * g0x - gy * g0y;
                gy = gx * g0y + gy * g0x;
                gx = nx;
                HostOp ph;
                memset(&ph, 0, sizeof(ph));
                ph.kind = OP_PHASE;
                ph.tq = -1;
                ph.cmask = bitq(h.tq);
                ph.cval = bitq(h.tq);
                if (bx != 1.0 || by != 0.0) {
                    ph.m[0] = bx;
                    ph.m[1] = by;
                    res.push_back(ph);
                }
                HostOp r;
                memset(&r, 0, sizeof(r));
                r.kind = OP_ROT;
                r.tq = h.tq;
                r.m[0] = c;
                r.m[1] = sm;
                res.push_back(r);
                if (ax != 1.0 || ay != 0.0) {
                    ph.m[0] = ax;
                    ph.m[1] = ay;
                    res.push_back(ph);
                }
                continue;
            }
        }
        res.push_back(h);
    }
    if (gx != 1.0 || gy != 0.0) {
        HostOp h;
        memset(&h, 0, sizeof(h));
        h.kind = OP_PHASE;
        h.tq = -1;
        h.m[0] = gx;
        h.m[1] = gy;
        res.push_back(h);
    }
    ops.swap(res);
    return xtail;
}

struct TileCfg {
    int n;    // qubits
    int apcLog; // 1 for fp32, 0 for fp64
    int L;    // low (contiguous) amplitude bits
    int kA;   // tile amplitude bits actually used
    int H;    // capacity of high qubits
    int maxOps; // ops per sweep (bounded by the shared-memory program area)
};

static TileCfg make_cfg(int n, int prec)
{
    TileCfg c;
    c.n = n;
    c.apcLog = (prec == 32) ? 1 : 0;
    const int kAmax = FUSED_KC + c.apcLog;
    c.kA = std::min(n, kAmax);
    c.L = std::min(FUSED_L, c.kA);
    if (n <= kAmax) {
        c.L = c.kA; // whole state is one tile
    }
    c.H = c.kA - c.L;
    c.maxOps = MAX_HOST_OPS;
    return c;
}

// Greedy, order-preserving selection with commutation-aware skipping.
//   fits(op)   : can the op be executed under the current resource set (may grow the set)
// Ops that are skipped block later ops that do not commute with them.
// Lazy diagonals (r2): a diagonal op commutes with everything except a non-diagonal op on one of its qubits, so it may be
// applied anywhere between its neighbours of that kind.  So a diagonal op is taken at once only when it costs
// nothing here (isFree: none of its qubits is a tile qubit -> per-tile scalar); otherwise it is DEFERRED without blocking
// anything, and pulled in right before the first taken non-diagonal op that acts on one of its qubits (so its phase joins
// the stage of that butterfly instead of costing a phase application of its own), or left for a later pass / sweep where it
// may be free.  When no non-diagonal op remains, the deferred ones are taken (progress, and no diagonal-only extra sweep).
template <typename FitFn, typename FreeFn>
static void greedy_select(std::vector<HostOp>& pending, std::vector<HostOp>& taken, size_t maxTake, size_t lookahead, FitFn fits,
    FreeFn isFree)
{
    uint64_t blockedT = 0, blockedD = 0;
    std::vector<char> gone(pending.size(), 0);
    std::vector<size_t> deferred;
    uint64_t deferredQ = 0;
    bool nonDiagLeft = false;
    size_t i = 0;
    for (; i < pending.size(); ++i) {
        const HostOp& op = pending[i];
        if (i >= lookahead || taken.size() >= maxTake) {
            break;
        }
        const uint64_t usesT = op.tq >= 0 ? bitq(op.tq) : 0;
        const uint64_t usesD = op.cmask;
        bool conflict = (usesT & (blockedT | blockedD)) || (usesD & blockedT);
        if (!conflict && op.kind == OP_PHASE && !isFree(op)) {
            deferred.push_back(i);
            deferredQ |= usesD;
            continue;
        }
        if (!conflict && !fits(op)) {
            conflict = true;
        }
        if (conflict) {
            blockedT |= usesT;
            blockedD |= usesD;
            nonDiagLeft = nonDiagLeft || op.kind != OP_PHASE;
        } else {
            if (usesT & deferredQ) {
                // the deferred diagonals on the target come first (they were unblocked when they were deferred)
                size_t w = 0;
                deferredQ = 0;
                for (size_t k = 0; k < deferred.size(); ++k) {
                    const size_t j = deferred[k];
                    if ((pending[j].cmask & usesT) && taken.size() + 1U < maxTake) {
                        taken.push_back(pending[j]);
                        gone[j] = 1;
                    } else {
                        deferred[w++] = j;
                        deferredQ |= pending[j].cmask;
                    }
                }
                deferred.resize(w);
                if (usesT & deferredQ) { // no room for a diagonal it needs: the op cannot run in this selection either
                    blockedT |= usesT;
                    blockedD |= usesD;
                    nonDiagLeft = true;
                    continue;
                }
            }
            taken.push_back(op);
            gone[i] = 1;
        }
    }
    for (size_t k = i; k < pending.size() && !nonDiagLeft; ++k) {
        nonDiagLeft = pending[k].kind != OP_PHASE;
    }
    if (!nonDiagLeft) {
        // only diagonal ops are left: take them now, in order
        for (size_t k = 0; k < pending.size() && taken.size() < maxTake; ++k) {
            if (!gone[k]) {
                taken.push_back(pending[k]);
                gone[k] = 1;
            }
        }
    }
    std::vector<HostOp> rest;
    rest.reserve(pending.size());
    for (size_t k = 0; k < pending.size(); ++k) {
        if (!gone[k]) {
            rest.push_back(pending[k]);
        }
    }
    pending.swap(rest);
}

struct PassPlan {
    std::vector<HostOp> ops;
    std::vector<int> regQ; // register qubits of this pass (excluding the implicit qubit 0 of fp32)
};
struct SweepPlan {
    std::vector<int> highQ; // ascending
    std::vector<PassPlan> passes;
    size_t nOps = 0;
};


// Count-only twin of greedy_select for a FIXED tile (no copies): how many of the first `lookahead` pending ops could run in
// a sweep whose tile qubits are `inTile`.
static size_t greedy_count(const std::vector<HostOp>& pending, size_t maxTake, size_t lookahead, uint64_t inTile)
{
    uint64_t blockedT = 0, blockedD = 0;
    size_t taken = 0;
    const size_t lim = std::min(pending.size(), lookahead);
    for (size_t i = 0; i < lim && taken < maxTake; ++i) {
        const HostOp& op = pending[i];
        const uint64_t usesT = op.tq >= 0 ? bitq(op.tq) : 0;
        const uint64_t usesD = op.cmask;
        if ((usesT & (blockedT | blockedD)) || (usesD & blockedT) || (usesT & ~inTile)) {
            blockedT |= usesT;
            blockedD |= usesD;
            if (!(inTile & ~(blockedT | blockedD))) {
                break; // every tile qubit is blocked: only stray diagonal gates could still be taken
            }
        } else {
            ++taken;
        }
    }
    return taken;
}

// hill-climbing rounds of the tile-qubit and register-qubit search.  On BASELINE's 30-qubit random circuit the search packs
// the 1800 gates into 38 sweeps instead of 51 (138 passes instead of 156) for ~3 ms of planning.
constexpr int SEARCH_ROUNDS = 2;

static void plan_sweep(std::vector<HostOp>& pending, const TileCfg& cfg, SweepPlan& sp)
{
    // ---- choose the tile's high qubits and the ops of this sweep ----
    uint64_t inTile = (cfg.L >= 64) ? ~0ULL : (bitq(cfg.L) - 1U);
    int freeHigh = cfg.H;
    std::vector<HostOp> sel;
    if (cfg.H > 0 && cfg.n > cfg.L + cfg.H) {
        // hill-climb on the set of high qubits: start from the order-of-first-use choice, swap one member at a time
        const uint64_t lowMask = inTile;
        uint64_t cur = lowMask;
        {
            int fh = cfg.H;
            uint64_t bT = 0, bD = 0;
            for (size_t i = 0; i < pending.size() && i < 2048 && fh > 0; ++i) {
                const HostOp& op = pending[i];
                const uint64_t uT = op.tq >= 0 ? bitq(op.tq) : 0, uD = op.cmask;
                if ((uT & (bT | bD)) || (uD & bT)) {
                    bT |= uT;
                    bD |= uD;
                } else if (uT & ~cur) {
                    cur |= uT;
                    --fh;
                }
            }
            for (int q = cfg.n - 1; q >= cfg.L && fh > 0; --q) {
                if (!(cur & bitq(q))) {
                    cur |= bitq(q);
                    --fh;
                }
            }
        }
        size_t best = greedy_count(pending, (size_t)cfg.maxOps, 2048, cur);
        for (int round = 0; round < SEARCH_ROUNDS; ++round) {
            uint64_t bestSet = cur;
            for (int h = cfg.L; h < cfg.n; ++h) {
                if (!(cur & bitq(h))) {
                    continue;
                }
                for (int c = cfg.L; c < cfg.n; ++c) {
                    if (cur & bitq(c)) {
                        continue;
                    }
                    const uint64_t cand = (cur & ~bitq(h)) | bitq(c);
                    const size_t got = greedy_count(pending, (size_t)cfg.maxOps, 2048, cand);
                    if (got > best) {
                        best = got;
                        bestSet = cand;
                    }
                }
            }
            if (bestSet == cur) {
                break;
            }
            cur = bestSet;
        }
        inTile = cur;
        freeHigh = 0;
    }
    greedy_select(
        pending, sel, (size_t)cfg.maxOps, 2048,
        [&](const HostOp& op) {
            if (op.tq < 0 || (inTile & bitq(op.tq))) {
                return true;
            }
            if (freeHigh > 0) {
                inTile |= bitq(op.tq);
                --freeHigh;
                return true;
            }
            return false;
        },
        [&](const HostOp& op) { return freeHigh == 0 && !(op.cmask & inTile); });
    sp.highQ.clear();
    for (int q = cfg.L; q < cfg.n; ++q) {
        if (inTile & bitq(q)) {
            sp.highQ.push_back(q);
        }
    }
    // pad the tile with arbitrary high qubits so that its size is fixed (top-down, any unused qubit)
    for (int q = cfg.n - 1; q >= cfg.L && (int)sp.highQ.size() < cfg.H; --q) {
        if (!(inTile & bitq(q))) {
            inTile |= bitq(q);
            sp.highQ.push_back(q);
        }
    }
    std::sort(sp.highQ.begin(), sp.highQ.end());
    // ---- split into passes by register capacity ----
    sp.passes.clear();
    sp.nOps = sel.size();
    while (!sel.empty() && (int)sp.passes.size() < MAX_PASS) {
        PassPlan pp;
        uint64_t regSet = cfg.apcLog ? 1ULL : 0ULL; // fp32: qubit 0 is always register-resident
        int freeReg = FUSED_RB;
        // same hill climbing for the pass's register qubits (targets must be register-resident, everything else rides along)
        const uint64_t fixed = regSet;
        uint64_t cur = fixed;
        int fr = FUSED_RB;
        uint64_t bT = 0, bD = 0;
        for (size_t i = 0; i < sel.size() && fr > 0; ++i) {
            const HostOp& op = sel[i];
            const uint64_t uT = op.tq >= 0 ? bitq(op.tq) : 0, uD = op.cmask;
            if ((uT & (bT | bD)) || (uD & bT)) {
                bT |= uT;
                bD |= uD;
            } else if (uT & ~cur) {
                cur |= uT;
                --fr;
            }
        }
        if (fr == 0) { // only worth searching when the pass is register-limited
            size_t best = greedy_count(sel, (size_t)cfg.maxOps, 4096, cur);
            for (int round = 0; round < SEARCH_ROUNDS; ++round) {
                uint64_t bestSet = cur;
                for (uint64_t hm = cur & ~fixed; hm; hm &= hm - 1U) {
                    const uint64_t hbit = hm & (~hm + 1U);
                    for (uint64_t cm = inTile & ~cur; cm; cm &= cm - 1U) {
                        const uint64_t cbit = cm & (~cm + 1U);
                        const uint64_t cand = (cur & ~hbit) | cbit;
                        const size_t got = greedy_count(sel, (size_t)cfg.maxOps, 4096, cand);
                        if (got > best) {
                            best = got;
                            bestSet = cand;
                        }
                    }
                }
                if (bestSet == cur) {
                    break;
                }
                cur = bestSet;
            }
            regSet = cur;
            freeReg = 0;
            for (uint64_t m = cur & ~fixed; m; m &= m - 1U) {
                pp.regQ.push_back(__builtin_ctzll(m));
            }
        }
        greedy_select(
            sel, pp.ops, (size_t)cfg.maxOps, 4096,
            [&](const HostOp& op) {
                if (op.tq < 0 || (regSet & bitq(op.tq))) {
                    return true;
                }
                if (freeReg > 0) {
                    regSet |= bitq(op.tq);
                    --freeReg;
                    pp.regQ.push_back(op.tq);
                    return true;
                }
                return false;
            },
            [&](const HostOp& op) { return !(op.cmask & inTile); });
        sp.passes.push_back(pp);
    }
    if (!sel.empty()) {
        // more passes than the descriptor holds: give the remainder back (order among them is preserved)
        sp.nOps -= sel.size();
        sel.insert(sel.end(), pending.begin(), pending.end());
        pending.swap(sel);
    }
}

// tile-local amplitude bit of a tile qubit
static int tile_bit(const TileCfg& cfg, const std::vector<int>& highQ, int q)
{
    if (q < cfg.L) {
        return q;
    }
    for (size_t h = 0; h < highQ.size(); ++h) {
        if (highQ[h] == q) {
            return cfg.L + (int)h;
        }
    }
    return -1;
}

// Encoded size limit of one sweep program plus its scratch (fits beside the 64 KB tile in shared memory with 2 CTAs/SM)
constexpr size_t MAX_PROG_BYTES_2CTA = 24576;

template <typename R>
static size_t encode_sweep(const SweepPlan& sp, const TileCfg& cfg, std::vector<unsigned char>& buf, size_t* scratchOut)
{
    const int kc = cfg.kA - cfg.apcLog;
    const int APC = 1 << cfg.apcLog;
    const int NCH = 1 << FUSED_RB;
    const int NA = NCH * APC;
    int JRN = 0;
    while ((1 << JRN) < NA) {
        ++JRN;
    }
    DevSweep ds;
    memset(&ds, 0, sizeof(ds));
    std::vector<DevOp<R>> dops;
    std::vector<DevOuterPhase<R>> outerList;
    std::vector<std::vector<DevOuterPhase<R>>> slotMembers; // table slots 1.. (register-bit phases of the STAGE ops)
    std::vector<DevMember<R>> memberList;                   // thread-level members of the STAGE ops
    std::vector<R> rotList;                                 // (c, s) of the STAGE ops' real rotations
    ds.nHigh = (int)sp.highQ.size();
    ds.lowAmpBits = cfg.L;
    ds.kc = kc;
    ds.nPass = (int)sp.passes.size();
    uint64_t tileMask = bitq(cfg.L) - 1U;
    for (int h = 0; h < ds.nHigh; ++h) {
        ds.highLow[h] = bitq(sp.highQ[h]) - 1U;
        ds.highPow[h] = bitq(sp.highQ[h]);
        tileMask |= bitq(sp.highQ[h]);
    }
    double scale = 1.0;
    for (int p = 0; p < ds.nPass; ++p) {
        const PassPlan& pp = sp.passes[p];
        DevPass& dp = ds.pass[p];
        // register chunk bits: targets first, then fill from the top with unused chunk bits
        std::vector<int> rb;
        uint32_t used = 0;
        for (int q : pp.regQ) {
            const int cb = tile_bit(cfg, sp.highQ, q) - cfg.apcLog;
            rb.push_back(cb);
            used |= 1U << cb;
        }
        for (int cb = kc - 1; cb >= 0 && (int)rb.size() < FUSED_RB; --cb) {
            if (!(used & (1U << cb))) {
                rb.push_back(cb);
                used |= 1U << cb;
            }
        }
        std::sort(rb.begin(), rb.end());
        // sub-block index bits: lanes first take one free bit from each bank class {0,3,6,9},{1,4,7,10},{2,5,8,11}
        std::vector<int> sb;
        uint32_t taken = used;
        for (int pcl = 0; pcl < 3; ++pcl) {
            for (int cand : { pcl, pcl + 3, pcl + 6, pcl + 9 }) {
                if (cand < kc && !(taken & (1U << cand))) {
                    sb.push_back(cand);
                    taken |= 1U << cand;
                    break;
                }
            }
        }
        for (int cb = 0; cb < kc; ++cb) {
            if (!(taken & (1U << cb))) {
                sb.push_back(cb);
                taken |= 1U << cb;
            }
        }
        dp.nsb = (int)sb.size();
        for (size_t i = 0; i < sb.size(); ++i) {
            dp.sbit[i] = (unsigned char)sb[i];
        }
        const uint32_t nSub = 1U << dp.nsb;
        dp.nIt = (int)std::max<uint32_t>(1U, nSub / (uint32_t)FUSED_NT);
        int tidBits = 0;
        while ((1 << tidBits) < FUSED_NT) {
            ++tidBits;
        }
        for (int it = 0; it < dp.nIt && it < 16; ++it) {
            uint32_t off = 0;
            for (int i = tidBits; i < dp.nsb; ++i) {
                if ((it >> (i - tidBits)) & 1) {
                    off |= 1U << sb[i];
                }
            }
            dp.itoffC[it] = (unsigned short)off;
        }
        // register chunk offsets and per-register-amplitude tile-local amplitude offsets
        uint32_t roffA[MAX_NA];
        uint32_t regAmpMask = cfg.apcLog ? 1U : 0U;
        for (int cb : rb) {
            regAmpMask |= 1U << (cb + cfg.apcLog);
        }
        for (int e = 0; e < NCH; ++e) {
            uint32_t off = 0;
            for (int b = 0; b < FUSED_RB; ++b) {
                if ((e >> b) & 1) {
                    off |= 1U << rb[b];
                }
            }
            dp.pswzB[e] = (unsigned short)(swz(off) << 4);
            {
                // the same chunk as a global amplitude offset relative to the tile base
                uint64_t g = 0;
                for (uint32_t ab = off << cfg.apcLog; ab; ab &= ab - 1U) {
                    const int tb = __builtin_ctz(ab);
                    g |= (tb < cfg.L) ? bitq(tb) : bitq(sp.highQ[tb - cfg.L]);
                }
                dp.goff[e] = g;
            }
            for (int w = 0; w < APC; ++w) {
                roffA[e * APC + w] = (off << cfg.apcLog) | (uint32_t)w;
            }
        }
        const uint32_t fullE = (uint32_t)((1ULL << NA) - 1ULL);
        auto reg_index = [&](int tb) {
            int jr = 0;
            for (int b = 0; b < tb; ++b) {
                if (regAmpMask & (1U << b)) {
                    ++jr;
                }
            }
            return jr;
        };
        // tile-local predicate of a host op: (lmask, lval) over tile amplitude bits
        auto local_pred = [&](const HostOp& hop, uint32_t& lmask, uint32_t& lval) {
            lmask = 0;
            lval = 0;
            for (uint64_t m = hop.cmask & tileMask; m; m &= m - 1U) {
                const int q = __builtin_ctzll(m);
                const int tb = tile_bit(cfg, sp.highQ, q);
                lmask |= 1U << tb;
                if (hop.cval & bitq(q)) {
                    lval |= 1U << tb;
                }
            }
        };
        // ---- open STAGE: per register bit J [phase][Hadamard], plus thread-uniform phases (group 0).  Its members are
        // diagonal except the butterflies, so a phase on bit J may join until the stage holds a butterfly on J; the stage is
        // emitted (closed) before the first single op that does not commute with its contents, or at the end of the pass.
        struct Stage {
            bool h[MAX_JR];
            bool isRot[MAX_JR];
            double rc[MAX_JR], rs[MAX_JR];
            std::vector<DevOuterPhase<R>> slot[MAX_JR]; // outer-only members of bit J's phase (per-tile product -> one table slot)
            std::vector<DevMember<R>> thr[MAX_JR + 1];  // group 0 = thread-uniform, 1 + J = bit J
            bool any;
        } st;
        auto stage_reset = [&]() {
            for (int b = 0; b < MAX_JR; ++b) {
                st.h[b] = false;
                st.isRot[b] = false;
                st.slot[b].clear();
            }
            for (int g = 0; g < MAX_JR + 1; ++g) {
                st.thr[g].clear();
            }
            st.any = false;
        };
        stage_reset();
        auto stage_slots = [&]() {
            int n = 0;
            for (int b = 0; b < MAX_JR; ++b) {
                n += st.slot[b].empty() ? 0 : 1;
            }
            return n;
        };
        auto stage_members = [&]() {
            size_t n = 0;
            for (int g = 0; g < MAX_JR + 1; ++g) {
                n += st.thr[g].size();
            }
            return n;
        };
        auto close_stage = [&]() {
            if (!st.any) {
                return;
            }
            DevOp<R> d;
            memset(&d, 0, sizeof(d));
            uint32_t hm = 0, sm = 0, rm = 0, cnts = 0;
            d.lmaskSb = (uint32_t)slotMembers.size() + 1U; // first table slot of this stage
            d.lvalSb = (uint32_t)memberList.size() | ((uint32_t)(rotList.size() / 2U) << 16); // first member | first rotation
            for (int g = 0; g < MAX_JR + 1; ++g) {
                cnts |= (uint32_t)st.thr[g].size() << (ST_CNT_BITS * g);
                memberList.insert(memberList.end(), st.thr[g].begin(), st.thr[g].end());
            }
            for (int b = 0; b < JRN; ++b) {
                if (st.h[b]) {
                    hm |= 1U << b;
                    if (st.isRot[b]) {
                        rm |= 1U << b;
                        rotList.push_back((R)st.rc[b]);
                        rotList.push_back((R)st.rs[b]);
                    }
                }
                if (!st.slot[b].empty()) {
                    sm |= 1U << b;
                    slotMembers.push_back(st.slot[b]);
                }
            }
            uint32_t act = hm | sm;
            for (int b = 0; b < MAX_JR; ++b) {
                if ((cnts >> (ST_CNT_BITS * (b + 1))) & ST_CNT_MASK) {
                    act |= 1U << b;
                }
            }
            d.code = OPC_STAGE;
            d.emask = hm | (sm << ST_SM_SHIFT) | (cnts ? (1U << ST_ANY_BIT) : 0U) | (act << ST_ACT_SHIFT) | (rm << ST_RM_SHIFT);
            memcpy(d.m, &cnts, sizeof(cnts));
            dops.push_back(d);
            stage_reset();
        };
        dp.opBegin = (int)dops.size();
        for (const HostOp& hop : pp.ops) {
            uint32_t lmask, lval;
            local_pred(hop, lmask, lval);
            const uint32_t lmr = lmask & regAmpMask, lvr = lval & regAmpMask;
            const int nreg = __builtin_popcount(lmr);
            if (hop.kind == OP_PHASE) {
                if (!(hop.cmask & tileMask) && outerList.size() < (size_t)MAX_OUTER) {
                    // every qubit of the predicate is outside the tile: uniform per tile, commutes with the whole sweep
                    DevOuterPhase<R> op;
                    memset(&op, 0, sizeof(op));
                    op.omask = hop.cmask;
                    op.oval = hop.cval;
                    op.ph[0] = (R)hop.m[0];
                    op.ph[1] = (R)hop.m[1];
                    outerList.push_back(op);
                    continue;
                }
                if (nreg <= 1 && lvr == lmr) {
                    // stage member: at most one register bit (value 1); thread bits and outer qubits anywhere
                    const int jr = nreg ? reg_index(__builtin_ctz(lmr)) : -1;
                    const bool threadPart = (lmask & ~regAmpMask) != 0;
                    const bool asSlot = nreg == 1 && !threadPart;
                    if (jr >= 0 && st.h[jr]) {
                        close_stage(); // the stage has a butterfly on this bit: the phase comes after it
                    }
                    auto fits = [&]() {
                        return asSlot ? (slotMembers.size() + (size_t)stage_slots() + (st.slot[jr].empty() ? 1U : 0U) + 2U < (size_t)MAX_SLOTS)
                                      : (st.thr[jr + 1].size() < (size_t)ST_CNT_MASK && memberList.size() + stage_members() + 1U < (size_t)MAX_MEMBERS);
                    };
                    if (!fits()) {
                        close_stage();
                    }
                    if (fits()) {
                        if (asSlot) {
                            DevOuterPhase<R> mem;
                            memset(&mem, 0, sizeof(mem));
                            mem.omask = hop.cmask & ~tileMask;
                            mem.oval = hop.cval & ~tileMask;
                            mem.ph[0] = (R)hop.m[0];
                            mem.ph[1] = (R)hop.m[1];
                            st.slot[jr].push_back(mem);
                        } else {
                            DevMember<R> mem;
                            memset(&mem, 0, sizeof(mem));
                            mem.omask = hop.cmask & ~tileMask;
                            mem.oval = hop.cval & ~tileMask;
                            mem.lmask = lmask & ~regAmpMask;
                            mem.lval = lval & ~regAmpMask;
                            mem.ph[0] = (R)hop.m[0];
                            mem.ph[1] = (R)hop.m[1];
                            st.thr[jr + 1].push_back(mem);
                        }
                        st.any = true;
                        continue;
                    }
                    // tables full: falls through to a single op
                }
            } else if (!hop.cmask && (hop.kind == OP_HAD || hop.kind == OP_ROT)) {
                // uncontrolled Hadamard / real rotation: butterfly of the stage (after the stage's phase on that bit)
                const int jr = reg_index(tile_bit(cfg, sp.highQ, hop.tq));
                if (st.h[jr] || rotList.size() / 2U + 8U >= 65535U) {
                    close_stage();
                }
                st.h[jr] = true;
                st.any = true;
                if (hop.kind == OP_ROT) {
                    st.isRot[jr] = true;
                    st.rc[jr] = hop.m[0];
                    st.rs[jr] = hop.m[1];
                } else {
                    scale *= hop.m[0];
                }
                continue;
            }
            // everything else is a single op, emitted at once: the open stage has to be closed first if the op does not
            // commute with its contents (target bit: any member; register-bit controls / phased register bits: a butterfly)
            {
                bool conflict = false;
                if (hop.tq >= 0) {
                    const int jt = reg_index(tile_bit(cfg, sp.highQ, hop.tq));
                    conflict = conflict || st.h[jt] || !st.slot[jt].empty() || !st.thr[jt + 1].empty();
                }
                for (uint32_t m = lmr; m; m &= m - 1U) {
                    conflict = conflict || st.h[reg_index(__builtin_ctz(m))];
                }
                if (conflict) {
                    close_stage();
                }
            }
            DevOp<R> d;
            memset(&d, 0, sizeof(d));
            d.omask = hop.cmask & ~tileMask;
            d.oval = hop.cval & ~tileMask;
            d.lmaskSb = lmask & ~regAmpMask;
            d.lvalSb = lval & ~regAmpMask;
            uint32_t em = 0;
            for (int e = 0; e < NA; ++e) {
                if ((roffA[e] & lmr) == lvr) {
                    em |= 1U << e;
                }
            }
            d.emask = em;
            const bool uncond = (em == fullE && d.lmaskSb == 0);
            for (int k = 0; k < 8; ++k) {
                d.m[k] = (R)hop.m[k];
            }
            uint32_t code = 0;
            if (hop.kind == OP_PHASE) {
                if (nreg == 2 && lvr == lmr) {
                    const int j = reg_index(__builtin_ctz(lmr)), k = reg_index(31 - __builtin_clz(lmr));
                    code = OPC_PH2 + (uint32_t)(k * (k - 1) / 2 + j);
                } else {
                    code = OPC_PHGEN;
                }
            } else {
                const uint32_t jr = (uint32_t)reg_index(tile_bit(cfg, sp.highQ, hop.tq));
                if (hop.kind == OP_XSWAP) {
                    code = K_XSWAP * 5U + jr;
                } else {
                    code = (uncond ? K_GEN_U : K_GEN_P) * 5U + jr;
                }
            }
            d.code = code | (d.lmaskSb ? CODE_HAS_SB : 0U) | (d.omask ? CODE_HAS_OUTER : 0U);
            if (code < OPC_PHGEN) {
                ds.needFull = 1;
            }
            dops.push_back(d);
        }
        close_stage();
        if (p == ds.nPass - 1 && (scale != 1.0 || !outerList.empty())) {
            DevOp<R> d;
            memset(&d, 0, sizeof(d));
            d.code = OPC_SCALE;
            dops.push_back(d);
        }
        dp.opEnd = (int)dops.size();
    }
    {
        auto lowRegBits = [&](const PassPlan& pp) {
            int cnt = 0;
            for (int q : pp.regQ) {
                const int cb = tile_bit(cfg, sp.highQ, q) - cfg.apcLog;
                if (cb >= 0 && cb < 3) {
                    ++cnt;
                }
            }
            return cnt;
        };
        // the first / last pass goes straight HBM <-> registers when at most one of its register bits is a chunk bit 0..2
        ds.directIn = (lowRegBits(sp.passes.front()) <= 1) ? 1 : 0;
        ds.directOut = (lowRegBits(sp.passes.back()) <= 1) ? 1 : 0;
    }
    ds.scale = scale;
    if (getenv("B200SV_FUSED_DEBUG")) {
        static const char* names[] = { "XSWAP", "GEN_U", "GEN_P" };
        for (int p = 0; p < ds.nPass; ++p) {
            fprintf(stderr, "  pass %d:", p);
            for (int o = ds.pass[p].opBegin; o < ds.pass[p].opEnd; ++o) {
                const uint32_t c = dops[o].code & 0xffU;
                const char* sfx = (dops[o].code & CODE_HAS_SB) ? "s" : "";
                const char* ofx = dops[o].omask ? "o" : "";
                if (c == OPC_STAGE) {
                    uint32_t cnts = 0;
                    memcpy(&cnts, dops[o].m, sizeof(cnts));
                    int nm = 0, nsl = 0;
                    for (int g = 0; g < MAX_JR + 1; ++g) {
                        nm += (int)((cnts >> (ST_CNT_BITS * g)) & ST_CNT_MASK);
                    }
                    for (int b = 0, sl = (int)dops[o].lmaskSb - 1; b < MAX_JR; ++b) {
                        if ((dops[o].emask >> ST_SM_SHIFT) & (1U << b)) {
                            nsl += (int)slotMembers[sl++].size();
                        }
                    }
                    fprintf(stderr, " STAGE(h%x,s%x:%d,t%d)", dops[o].emask & ST_MASK, (dops[o].emask >> ST_SM_SHIFT) & ST_MASK, nsl, nm);
                } else if (c == OPC_SCALE) {
                    fprintf(stderr, " SCALE");
                } else if (c == OPC_PHGEN) {
                    fprintf(stderr, " PHGEN%s%s", sfx, ofx);
                } else if (c >= OPC_PH2) {
                    fprintf(stderr, " PH2.%u%s%s", c - OPC_PH2, sfx, ofx);
                } else {
                    fprintf(stderr, " %s.%u%s%s", names[c / 5U], c % 5U, sfx, ofx);
                }
            }
            fprintf(stderr, "\n");
        }
        fprintf(stderr, "  sweep: %d ops, %d outer phases, %d thread members, directIn %d, directOut %d\n", (int)dops.size(),
            (int)outerList.size(), (int)memberList.size(), ds.directIn, ds.directOut);
    }
    ds.hasScale = (scale != 1.0 || !outerList.empty()) ? 1 : 0;
    ds.nOps = (int)dops.size();
    ds.nOuter = (int)outerList.size();
    // table slots: slot 0 = the outer-only phases (tile scalar), then one slot per (DIAG op, register bit)
    ds.nSlots = 1 + (int)slotMembers.size();
    {
        const int lcb = cfg.L - cfg.apcLog;
        const size_t rows = (size_t)1 << (kc > lcb ? kc - lcb : 0);
        ds.scratchBytes =
            (int)((rows * 8U + (size_t)4 * (size_t)ds.nSlots * sizeof(R) + (size_t)16 * memberList.size() +
                      (size_t)2 * (size_t)ds.nPass * (size_t)FUSED_NT + 15U) & ~(size_t)15U); // + per-(pass, thread) sub-block bases
    }
    ds.nMem = (int)memberList.size();
    ds.slotBeg[0] = 0;
    ds.slotBeg[1] = (unsigned short)outerList.size();
    for (size_t k = 0; k < slotMembers.size(); ++k) {
        outerList.insert(outerList.end(), slotMembers[k].begin(), slotMembers[k].end());
        ds.slotBeg[k + 2] = (unsigned short)outerList.size();
    }
    const size_t opsBytes = ((dops.size() * sizeof(DevOp<R>)) + 15U) & ~(size_t)15U;
    const size_t outerBytes = ((outerList.size() * sizeof(DevOuterPhase<R>)) + 15U) & ~(size_t)15U;
    const size_t memBytes = memberList.size() * sizeof(DevMember<R>); // multiple of 16
    ds.outerOff = (int)(sizeof(DevSweep) + opsBytes);
    ds.memOff = (int)(sizeof(DevSweep) + opsBytes + outerBytes);
    const size_t rotBytes = (rotList.size() * sizeof(R) + 15U) & ~(size_t)15U;
    ds.rotOff = (int)(sizeof(DevSweep) + opsBytes + outerBytes + memBytes);
    ds.nRot = (int)(rotList.size() / 2U);
    const size_t start = buf.size();
    size_t bytes = ((sizeof(DevSweep) + opsBytes + outerBytes + memBytes + rotBytes) + 15U) & ~(size_t)15U;
    if (scratchOut) {
        *scratchOut = (size_t)ds.scratchBytes;
    }
    if (dops.size() > (size_t)MAX_OPS || outerList.size() > 60000U) {
        bytes = (size_t)1 << 30; // does not fit the descriptor: the caller retries with a smaller window
        return bytes;
    }
    buf.resize(start + bytes, 0);
    memcpy(buf.data() + start, &ds, sizeof(ds));
    if (!dops.empty()) {
        memcpy(buf.data() + start + sizeof(DevSweep), dops.data(), dops.size() * sizeof(DevOp<R>));
    }
    if (!outerList.empty()) {
        memcpy(buf.data() + start + ds.outerOff, outerList.data(), outerList.size() * sizeof(DevOuterPhase<R>));
    }
    if (!memberList.empty()) {
        memcpy(buf.data() + start + ds.memOff, memberList.data(), memBytes);
    }
    if (!rotList.empty()) {
        memcpy(buf.data() + start + ds.rotOff, rotList.data(), rotList.size() * sizeof(R));
    }
    return bytes;
}

// Plan + encode ONE sweep from the head of `pending`.  Planning works on a bounded window (the scheduler never looks
// further ahead than that), and retries with fewer ops if the encoded program would not fit beside the tile.
constexpr size_t PLAN_WINDOW = 1024;
static int plan_and_encode(std::vector<HostOp>& pending, const TileCfg& cfg0, int prec, std::vector<unsigned char>& buf, size_t* bytesOut,
    size_t* scratchOut, size_t* nOpsOut, int* nPassOut)
{
    const size_t wsz = std::min(pending.size(), PLAN_WINDOW);
    TileCfg cfg = cfg0;
    for (;;) {
        std::vector<HostOp> window(pending.begin(), pending.begin() + wsz);
        SweepPlan sp;
        plan_sweep(window, cfg, sp);
        if (!sp.nOps) {
            set_error("fused scheduler made no progress");
            return B200SV_ESTATE;
        }
        const size_t mark = buf.size();
        size_t scratch = 0;
        const size_t bytes =
            (prec == 32) ? encode_sweep<float>(sp, cfg, buf, &scratch) : encode_sweep<double>(sp, cfg, buf, &scratch);
        if (bytes + scratch > MAX_PROG_BYTES_2CTA) {
            if (cfg.maxOps <= 4) {
                set_error("fused sweep program does not fit");
                return B200SV_ESTATE;
            }
            buf.resize(mark);
            cfg.maxOps = cfg.maxOps * 3 / 4;
            continue;
        }
        // commit: the window's leftovers go back in front of the untouched tail
        window.insert(window.end(), pending.begin() + wsz, pending.end());
        pending.swap(window);
        *bytesOut = bytes;
        *scratchOut = scratch;
        *nOpsOut = sp.nOps;
        *nPassOut = (int)sp.passes.size();
        return B200SV_OK;
    }
}

// One encoded sweep inside the flush's program buffer
struct Seg {
    size_t off, bytes, scratch, nops;
    int npass;
};

// Plans and encodes every sweep of a flush: `pending` is consumed.
static int plan_list(std::vector<HostOp>& pending, const TileCfg& cfg, int prec, std::vector<unsigned char>& buf, std::vector<Seg>& segs)
{
    while (!pending.empty()) {
        const size_t off = buf.size();
        size_t bytes = 0, scratch = 0, nops = 0;
        int npass = 0;
        SV_TRY(plan_and_encode(pending, cfg, prec, buf, &bytes, &scratch, &nops, &npass));
        segs.push_back({ off, bytes, scratch, nops, npass });
        if (getenv("B200SV_FUSED_DEBUG")) {
            fprintf(stderr, "  program %zu B + scratch %zu B\n", bytes, scratch);
        }
    }
    return B200SV_OK;
}

// per-state program arena (device + pinned host), guarded by an event
struct Arena {
    unsigned char* dev = nullptr;
    unsigned char* host = nullptr;
    size_t cap = 0;
    cudaEvent_t done = nullptr;
    bool pending = false;
};
// Registry state -> arena.  The arenas live on the heap (stable addresses): QPager drives its page engines from several
// host threads, so one thread may register or release a state while another still holds its own arena pointer.
static std::vector<std::pair<State*, std::unique_ptr<Arena>>>& arenas()
{
    static std::vector<std::pair<State*, std::unique_ptr<Arena>>> a;
    return a;
}
static std::mutex& arena_mutex()
{
    static std::mutex m;
    return m;
}
static Arena* get_arena(State* s)
{
    std::lock_guard<std::mutex> lk(arena_mutex());
    for (auto& kv : arenas()) {
        if (kv.first == s) {
            return kv.second.get();
        }
    }
    arenas().emplace_back(s, std::unique_ptr<Arena>(new Arena()));
    return arenas().back().second.get();
}
void fused_release(State* s)
{
    std::unique_ptr<Arena> mine;
    {
        std::lock_guard<std::mutex> lk(arena_mutex());
        auto& v = arenas();
        for (size_t i = 0; i < v.size(); ++i) {
            if (v[i].first == s) {
                mine = std::move(v[i].second);
                v.erase(v.begin() + i);
                break;
            }
        }
    }
    if (mine) {
        if (mine->dev) {
            cudaFree(mine->dev);
        }
        if (mine->host) {
            cudaFreeHost(mine->host);
        }
        if (mine->done) {
            cudaEventDestroy(mine->done);
        }
    }
}

bool fused_accepts(const State* s, const GateOp&) { return s->nq >= 5 && s->nq <= 62; }

template <typename R, int VAR, bool PULL = false>
static int launch_sweep_v(State* s, const unsigned char* dprog, uint32_t progBytes, uint32_t scratchBytes, uint64_t nTiles)
{
    auto kern = k_fused_sweep<R, VAR, PULL>;
    const size_t shm = ((size_t)16 << FUSED_KC) + progBytes + scratchBytes;
    static std::atomic<unsigned long long> attr_set_mask{ 0 }; // per device: the attribute is per-context
    if (!(attr_set_mask.load() & (1ULL << s->dev))) {
        SV_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(((size_t)16 << FUSED_KC) + MAX_PROG_BYTES_2CTA)));
        attr_set_mask.fetch_or(1ULL << s->dev);
    }
    const uint64_t maxGrid = (uint64_t)sm_count(s->dev) * FUSED_MINB;
    const unsigned grid = (unsigned)std::min<uint64_t>(nTiles, maxGrid);
    kern<<<grid, FUSED_NT, shm, s->stream>>>(reinterpret_cast<typename Cx<R>::type*>(s->amps), dprog, progBytes, nTiles,
        PULL ? s->pull : PullArgs{});
    SV_CUDA(cudaGetLastError());
    if (PULL) {
        s->amps = s->pull.out; // the rest of the flush (and everything after it) works in place on the new page
        s->pullPending = false;
    }
    return B200SV_OK;
}

template <typename R>
static int launch_sweep(State* s, const unsigned char* dprog, uint32_t progBytes, uint32_t scratchBytes, uint64_t nTiles, int var)
{
    // var: 0 = light (STAGE / phase ops, Hadamard butterflies only), 1 = light + rotation stages, 2 = full (+ swap / general-matrix ops)
    return var == 2 ? launch_sweep_v<R, 2>(s, dprog, progBytes, scratchBytes, nTiles)
                    : (var == 1 ? launch_sweep_v<R, 1>(s, dprog, progBytes, scratchBytes, nTiles)
                                : launch_sweep_v<R, 0>(s, dprog, progBytes, scratchBytes, nTiles));
}

int fused_flush(State* s)
{
    if (s->queue.empty()) {
        return s->pullPending ? launch_pull_gather(s) : B200SV_OK;
    }
    if (!s->amps) {
        s->queue.clear();
        return B200SV_OK;
    }
    std::vector<HostOp> pending;
    const uint64_t xtail = lower_queue(s->queue, pending);
    const size_t nGates = s->queue.size();
    const TileCfg cfg = make_cfg(s->nq, s->prec);
    // build every sweep of this flush (nothing is launched before the whole flush is planned: a planner failure leaves the state as it was)
    std::vector<unsigned char> buf;
    std::vector<Seg> segs;
    SV_TRY(plan_list(pending, cfg, s->prec, buf, segs));
    s->queue.clear();
    // A pending re-page rides on the first sweep when there is one; otherwise it is a plain gather.
    if (s->pullPending && segs.empty()) {
        SV_TRY(launch_pull_gather(s));
    }
    if (segs.empty()) {
        return xtail ? launch_xmask(s, xtail) : B200SV_OK;
    }
    Arena* ar = get_arena(s);
    if (!ar->done) {
        SV_CUDA(cudaEventCreateWithFlags(&ar->done, cudaEventDisableTiming));
    }
    const uint64_t nTiles = s->dim() >> cfg.kA;
    if (ar->pending) {
        SV_CUDA(cudaEventSynchronize(ar->done));
        ar->pending = false;
    }
    if (ar->cap < buf.size()) {
        if (ar->dev) {
            cudaFree(ar->dev);
            cudaFreeHost(ar->host);
        }
        ar->cap = std::max<size_t>(buf.size() * 2, 1 << 20);
        SV_CUDA(cudaMalloc(&ar->dev, ar->cap));
        SV_CUDA(cudaMallocHost(&ar->host, ar->cap));
    }
    memcpy(ar->host, buf.data(), buf.size());
    SV_CUDA(cudaMemcpyAsync(ar->dev, ar->host, buf.size(), cudaMemcpyHostToDevice, s->stream));
    for (size_t i = 0; i < segs.size(); ++i) {
        const unsigned char* dp = ar->dev + segs[i].off;
        const uint32_t pb = (uint32_t)segs[i].bytes, sb = (uint32_t)segs[i].scratch;
        const DevSweep* dsw = reinterpret_cast<const DevSweep*>(buf.data() + segs[i].off);
        const bool full = dsw->needFull != 0;
        const int var = full ? 2 : (dsw->nRot ? 1 : 0);
        if (s->pullPending) {
            // (i == 0) the re-page rides on this sweep: the full variant
            if (s->prec == 32) {
                SV_TRY((launch_sweep_v<float, 2, true>(s, dp, pb, sb, nTiles)));
            } else {
                SV_TRY((launch_sweep_v<double, 2, true>(s, dp, pb, sb, nTiles)));
            }
            s->stats.pull_sweeps++;
        } else if (s->prec == 32) {
            SV_TRY(launch_sweep<float>(s, dp, pb, sb, nTiles, var));
        } else {
            SV_TRY(launch_sweep<double>(s, dp, pb, sb, nTiles, var));
        }
        s->stats.kernel_launches++;
        s->stats.fused_sweeps++;
        s->stats.bytes_swept += 2ULL * s->dim() * s->amp_bytes();
    }
    s->stats.fused_gates += nGates;
    SV_CUDA(cudaEventRecord(ar->done, s->stream));
    ar->pending = true;
    if (xtail) {
        SV_TRY(launch_xmask(s, xtail));
    }
    return B200SV_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Host emulation of the sweep programs (TEST HOOK, never on the engine's path): runs the planner + encoder on a gate
// list and then interprets every encoded sweep on a HOST state vector, following the device kernel table by table —
// tile base (push-apart), active-op ballots, outer/DIAG phase slots, per-pass thread -> sub-block map (sbit / itoffC),
// register-chunk tables (goff for the HBM side, swizzled pswzB for the smem tile), staged vs direct first/last pass and
// the op semantics of exec_op.  `pytest -m "not gpu"` uses it to check scheduler and encoder against the oracle
// without a device (tests/test_fused_emulation.py).
// ---------------------------------------------------------------------------------------------------------
template <typename R> struct EmuC {
    R x, y;
};
template <typename R> static inline EmuC<R> emu_mul(EmuC<R> a, R px, R py) { return EmuC<R>{ a.x * px - a.y * py, a.x * py + a.y * px }; }

template <typename R>
static void emu_exec_op(std::vector<EmuC<R>>& a, const DevOp<R>& op, uint32_t xsb, const R* tileScale, int NA,
    const DevMember<R>* members, const uint2* eff, const R* rotTab)
{
    const uint32_t code = op.code, emask = op.emask, lmaskSb = op.lmaskSb, lvalSb = op.lvalSb;
    bool tp = true;
    if (code & CODE_HAS_SB) {
        tp = (xsb & lmaskSb) == lvalSb;
    }
    const uint32_t em = tp ? emask : 0U;
    const uint32_t c = code & 0xffU;
    auto had = [&](int J) {
        for (int e = 0; e < NA; ++e) {
            if (!(e & (1 << J))) {
                const EmuC<R> x = a[e], y = a[e | (1 << J)];
                a[e] = EmuC<R>{ x.x + y.x, x.y + y.y };
                a[e | (1 << J)] = EmuC<R>{ x.x - y.x, x.y - y.y };
            }
        }
    };
    auto phase_reg = [&](int J, R px, R py) {
        for (int e = 0; e < NA; ++e) {
            if (e & (1 << J)) {
                a[e] = emu_mul(a[e], px, py);
            }
        }
    };
    if (c == OPC_STAGE) {
        const uint32_t hm = emask & ST_MASK, sm = (emask >> ST_SM_SHIFT) & ST_MASK, rm = (emask >> ST_RM_SHIFT) & ST_MASK;
        uint32_t slot = lmaskSb, mk = lvalSb & 0xffffU, ri = lvalSb >> 16, cnts = 0;
        if (emask & (1U << ST_ANY_BIT)) {
            memcpy(&cnts, op.m, sizeof(cnts));
        }
        auto run_members = [&](uint32_t cN, R& px, R& py) {
            for (uint32_t k = 0; k < cN; ++k, ++mk) {
                if ((xsb & eff[mk].x) == eff[mk].y) {
                    const R qx = members[mk].ph[0], qy = members[mk].ph[1];
                    const R nx = px * qx - py * qy;
                    py = px * qy + py * qx;
                    px = nx;
                }
            }
        };
        {
            R px = (R)1, py = (R)0;
            run_members(cnts & ST_CNT_MASK, px, py);
            if (px != (R)1 || py != (R)0) {
                for (int e = 0; e < NA; ++e) {
                    a[e] = emu_mul(a[e], px, py);
                }
            }
        }
        for (int J = 0; (1 << J) < NA; ++J) {
            const uint32_t cN = (cnts >> (ST_CNT_BITS * (J + 1))) & ST_CNT_MASK;
            R px = (R)1, py = (R)0;
            if ((sm >> J) & 1U) {
                px = tileScale[2 * slot];
                py = tileScale[2 * slot + 1];
                ++slot;
            }
            run_members(cN, px, py);
            if (px != (R)1 || py != (R)0) {
                phase_reg(J, px, py);
            }
            if ((hm >> J) & 1U) {
                if ((rm >> J) & 1U) {
                    const R c = rotTab[2 * ri], sn = rotTab[2 * ri + 1];
                    ++ri;
                    for (int e = 0; e < NA; ++e) {
                        if (!(e & (1 << J))) {
                            const EmuC<R> x = a[e], y = a[e | (1 << J)];
                            a[e] = EmuC<R>{ c * x.x - sn * y.x, c * x.y - sn * y.y };
                            a[e | (1 << J)] = EmuC<R>{ sn * x.x + c * y.x, sn * x.y + c * y.y };
                        }
                    }
                } else {
                    had(J);
                }
            }
        }
        return;
    }
    if (c == OPC_SCALE) {
        for (int e = 0; e < NA; ++e) {
            a[e] = emu_mul(a[e], tileScale[0], tileScale[1]);
        }
        return;
    }
    if (c == OPC_PHGEN) {
        for (int e = 0; e < NA; ++e) {
            if ((em >> e) & 1U) {
                a[e] = emu_mul(a[e], op.m[0], op.m[1]);
            }
        }
        return;
    }
    if (c >= OPC_PH2) {
        int k = 1;
        while ((k + 1) * k / 2 <= (int)(c - OPC_PH2)) {
            ++k;
        }
        const int j = (int)(c - OPC_PH2) - k * (k - 1) / 2;
        if (tp) {
            for (int e = 0; e < NA; ++e) {
                if ((e & (1 << j)) && (e & (1 << k))) {
                    a[e] = emu_mul(a[e], op.m[0], op.m[1]);
                }
            }
        }
        return;
    }
    const uint32_t kind = c / 5U;
    const int J = (int)(c % 5U);
    const R* m = op.m;
    switch (kind) {
    case K_XSWAP:
        for (int e = 0; e < NA; ++e) {
            if (!(e & (1 << J)) && ((em >> e) & 1U)) {
                std::swap(a[e], a[e | (1 << J)]);
            }
        }
        break;
    case K_GEN_U:
    case K_GEN_P:
        for (int e = 0; e < NA; ++e) {
            if (!(e & (1 << J)) && (kind == K_GEN_U || ((em >> e) & 1U))) {
                const EmuC<R> x = a[e], y = a[e | (1 << J)];
                const EmuC<R> x0 = emu_mul(x, m[0], m[1]), y1 = emu_mul(y, m[2], m[3]);
                const EmuC<R> x2 = emu_mul(x, m[4], m[5]), y3 = emu_mul(y, m[6], m[7]);
                a[e] = EmuC<R>{ x0.x + y1.x, x0.y + y1.y };
                a[e | (1 << J)] = EmuC<R>{ x2.x + y3.x, x2.y + y3.y };
            }
        }
        break;
    default:
        break;
    }
}

// `pull` (first sweep of a flush with a pending re-page): reads go through the source pages with the device's pull_src mapping,
// writes go to `psi` (the out page)
template <typename R> static EmuC<R> emu_pull_load(const PullArgs& pa, uint64_t i)
{
    unsigned r = 0;
    for (int b = 0; b < pa.k; ++b) {
        r |= (unsigned)((i >> pa.vb[b]) & 1ULL) << b;
    }
    return reinterpret_cast<const EmuC<R>*>(pa.peers[r])[(i & ~pa.vmask) | pa.rankDep];
}

template <typename R>
static void emulate_sweep(const unsigned char* prog, EmuC<R>* psi, int nq, const TileCfg& cfg, const PullArgs* pull = nullptr)
{
    const DevSweep& sw = *reinterpret_cast<const DevSweep*>(prog);
    const DevOp<R>* ops = reinterpret_cast<const DevOp<R>*>(prog + sizeof(DevSweep));
    const DevOuterPhase<R>* outer = reinterpret_cast<const DevOuterPhase<R>*>(prog + sw.outerOff);
    const int APC = 1 << cfg.apcLog, NCH = 1 << FUSED_RB, NA = NCH * APC, NT = FUSED_NT;
    const int kc = sw.kc;
    const uint32_t nChunk = 1U << kc;
    const int lcb = sw.lowAmpBits - cfg.apcLog;
    const uint32_t colMask = (1U << lcb) - 1U;
    const uint32_t nRows = nChunk >> lcb;
    std::vector<uint64_t> rowOff(nRows);
    for (uint32_t r = 0; r < nRows; ++r) {
        uint64_t off = 0;
        for (int h = 0; h < sw.nHigh; ++h) {
            if ((r >> h) & 1U) {
                off |= sw.highPow[h];
            }
        }
        rowOff[r] = off;
    }
    const uint32_t nSub = nChunk >> FUSED_RB;
    const uint64_t nTiles = (1ULL << nq) >> cfg.kA;
    std::vector<EmuC<R>> tile((size_t)nChunk * APC); // indexed by swizzled chunk slot
    std::vector<R> tab((size_t)2 * std::max(1, sw.nSlots));
    std::vector<EmuC<R>> a((size_t)NA);
    const DevMember<R>* members = reinterpret_cast<const DevMember<R>*>(prog + sw.memOff);
    const R* rotTab = reinterpret_cast<const R*>(prog + sw.rotOff);
    std::vector<uint2> eff((size_t)std::max(1, sw.nMem));
    for (uint64_t t = 0; t < nTiles; ++t) {
        uint64_t base = t << sw.lowAmpBits;
        for (int h = 0; h < sw.nHigh; ++h) {
            const uint64_t lo = base & sw.highLow[h];
            base = ((base ^ lo) << 1) | lo;
        }
        EmuC<R>* const tilePsi = psi + base;
        // preamble: ballots, tile scalar, DIAG slots
        std::vector<bool> act((size_t)std::max(1, sw.nOps));
        for (int o = 0; o < sw.nOps; ++o) {
            act[o] = (base & ops[o].omask) == ops[o].oval;
        }
        {
            double fx = 1.0, fy = 0.0;
            for (int i = 0; i < sw.nOuter; ++i) {
                if ((base & outer[i].omask) == outer[i].oval) {
                    const double nx = fx * (double)outer[i].ph[0] - fy * (double)outer[i].ph[1];
                    fy = fx * (double)outer[i].ph[1] + fy * (double)outer[i].ph[0];
                    fx = nx;
                }
            }
            tab[0] = (R)(fx * sw.scale);
            tab[1] = (R)(fy * sw.scale);
        }
        for (int sl = 1; sl < sw.nSlots; ++sl) {
            double fx = 1.0, fy = 0.0;
            for (int i = sw.slotBeg[sl]; i < sw.slotBeg[sl + 1]; ++i) {
                if ((base & outer[i].omask) == outer[i].oval) {
                    const double nx = fx * (double)outer[i].ph[0] - fy * (double)outer[i].ph[1];
                    fy = fx * (double)outer[i].ph[1] + fy * (double)outer[i].ph[0];
                    fx = nx;
                }
            }
            tab[2 * sl] = (R)fx;
            tab[2 * sl + 1] = (R)fy;
        }
        for (int i = 0; i < sw.nMem; ++i) {
            const bool ok = (base & members[i].omask) == members[i].oval;
            eff[(size_t)i] = ok ? make_uint2(members[i].lmask, members[i].lval) : make_uint2(0U, 1U);
        }
        if (!sw.directIn) {
            for (uint32_t c = 0; c < nChunk; ++c) {
                for (int w = 0; w < APC; ++w) {
                    const uint64_t off = rowOff[c >> lcb] + (uint64_t)(c & colMask) * APC + w;
                    tile[(size_t)swz(c) * APC + w] = pull ? emu_pull_load<R>(*pull, base + off) : tilePsi[off];
                }
            }
        }
        for (int p = 0; p < sw.nPass; ++p) {
            const DevPass& ps = sw.pass[p];
            const bool fromGlobal = (p == 0) && sw.directIn, toGlobal = (p == sw.nPass - 1) && sw.directOut;
            for (int tid = 0; tid < NT; ++tid) {
                uint32_t dep = 0;
                const int nb = ps.nsb < 8 ? ps.nsb : 8;
                for (int i = 0; i < nb; ++i) {
                    dep |= (((uint32_t)tid >> i) & 1U) << ps.sbit[i];
                }
                for (int it = 0; it < ps.nIt; ++it) {
                    if ((uint32_t)(it * NT + tid) >= nSub) {
                        break;
                    }
                    const uint32_t sbc = dep | ps.itoffC[it];
                    const uint32_t swb = swz(sbc) << 4;
                    EmuC<R>* const gsub = tilePsi + rowOff[sbc >> lcb] + (uint64_t)(sbc & colMask) * APC;
                    for (int e = 0; e < NCH; ++e) {
                        for (int w = 0; w < APC; ++w) {
                            a[(size_t)e * APC + w] = !fromGlobal
                                ? tile[(size_t)((swb ^ ps.pswzB[e]) >> 4) * APC + w]
                                : (pull ? emu_pull_load<R>(*pull, (uint64_t)(gsub - psi) + ps.goff[e] + w) : gsub[ps.goff[e] + w]);
                        }
                    }
                    const uint32_t xsb = sbc * (uint32_t)APC;
                    for (int o = ps.opBegin; o < ps.opEnd; ++o) {
                        if (act[o]) {
                            emu_exec_op<R>(a, ops[o], xsb, tab.data(), NA, members, eff.data(), rotTab);
                        }
                    }
                    for (int e = 0; e < NCH; ++e) {
                        for (int w = 0; w < APC; ++w) {
                            if (toGlobal) {
                                gsub[ps.goff[e] + w] = a[(size_t)e * APC + w];
                            } else {
                                tile[(size_t)((swb ^ ps.pswzB[e]) >> 4) * APC + w] = a[(size_t)e * APC + w];
                            }
                        }
                    }
                }
            }
        }
        if (!sw.directOut) {
            for (uint32_t c = 0; c < nChunk; ++c) {
                for (int w = 0; w < APC; ++w) {
                    tilePsi[rowOff[c >> lcb] + (uint64_t)(c & colMask) * APC + w] = tile[(size_t)swz(c) * APC + w];
                }
            }
        }
    }
}

int fused_emulate(int n_qubits, int precision, const std::vector<GateOp>& q, void* host_state, const PullArgs* pull)
{
    std::vector<HostOp> pending;
    const uint64_t xtail = lower_queue(q, pending);
    const TileCfg cfg = make_cfg(n_qubits, precision);
    std::vector<unsigned char> buf;
    std::vector<Seg> segs;
    SV_TRY(plan_list(pending, cfg, precision, buf, segs));
    if (pull && segs.empty()) { // launch_pull_gather on the device
        const uint64_t dim = 1ULL << n_qubits;
        for (uint64_t i = 0; i < dim; ++i) {
            if (precision == 32) {
                reinterpret_cast<EmuC<float>*>(host_state)[i] = emu_pull_load<float>(*pull, i);
            } else {
                reinterpret_cast<EmuC<double>*>(host_state)[i] = emu_pull_load<double>(*pull, i);
            }
        }
        pull = nullptr;
    }
    for (const Seg& sg : segs) {
        if (precision == 32) {
            emulate_sweep<float>(buf.data() + sg.off, reinterpret_cast<EmuC<float>*>(host_state), n_qubits, cfg, pull);
        } else {
            emulate_sweep<double>(buf.data() + sg.off, reinterpret_cast<EmuC<double>*>(host_state), n_qubits, cfg, pull);
        }
        pull = nullptr; // only the first sweep carries the re-page
    }
    if (xtail) { // the trailing XMask sweep (launch_xmask on the device)
        const uint64_t dim = 1ULL << n_qubits;
        const size_t ab = (precision == 32) ? 8 : 16;
        unsigned char* st = reinterpret_cast<unsigned char*>(host_state);
        unsigned char tmp[16];
        for (uint64_t i = 0; i < dim; ++i) {
            const uint64_t j = i ^ xtail;
            if (i < j) {
                memcpy(tmp, st + i * ab, ab);
                memcpy(st + i * ab, st + j * ab, ab);
                memcpy(st + j * ab, tmp, ab);
            }
        }
    }
    return B200SV_OK;
}

// what a flush of this gate list would launch: sweeps, passes, device ops (host only; scripts/shard_sweep_count.py)
int fused_plan_gates(int n_qubits, int precision, const std::vector<GateOp>& q, int* n_sweeps, int* n_passes, int* n_ops)
{
    std::vector<HostOp> pending;
    (void)lower_queue(q, pending);
    const TileCfg cfg = make_cfg(n_qubits, precision);
    int sweeps = 0, passes = 0, ops = 0;
    std::vector<unsigned char> buf;
    while (!pending.empty()) {
        size_t bytes = 0, nops = 0, scratch = 0;
        int npass = 0;
        buf.clear();
        SV_TRY(plan_and_encode(pending, cfg, precision, buf, &bytes, &scratch, &nops, &npass));
        ++sweeps;
        passes += npass;
        ops += (int)nops;
    }
    *n_sweeps = sweeps;
    *n_passes = passes;
    *n_ops = ops;
    return B200SV_OK;
}

} // namespace b200sv
