/* b200sv.h — C ABI of the H100 (sm_90a) state-vector core (libb200sv.so).
 *
 * This is the drop-in boundary for the QEngine gate hot path of unitaryfoundation/qrack: every entry
 * point below is what a `Qrack::QEngine` subclass (the `QEngineCUDA` slot, reference
 * include/qengine_cuda.hpp:280-284, selected by include/qfactory.hpp:80,128,172,237) needs to forward
 * one of its pure virtuals to.  The C++ adapter that does exactly that against the reference's own
 * headers lives in dropin/ (see INTEGRATION.md); qrack_b200/qengine.py is the same adapter in Python
 * over ctypes.  Each function cites the reference interface it replaces.
 *
 * Conventions
 *  - extern "C", plain pointers and sizes, no C++/torch types.  Every call returns B200SV_OK (0) or a
 *    negative error code; b200sv_last_error() returns the message of the calling thread's last failure
 *    (the adapter turns B200SV_EINVAL into std::invalid_argument, B200SV_ENOMEM into Qrack::bad_alloc,
 *    everything else into std::runtime_error — reference conventions, SURVEY.md §8b.3).
 *  - A state has 2^n amplitudes, interleaved (re,im), little-endian qubit order: bit k of the index is
 *    qubit k (reference include/statevector.hpp:94,153-168).  precision 32 = float2, 64 = double2.
 *    Host amplitude/probability buffers are in the state's precision; all scalars cross as double.
 *  - A state may be "zero" (no device buffer, all amplitudes 0) exactly like QEngineCPU's null stateVec
 *    (reference src/qengine/state.cpp:20-24 CHECK_ZERO_SKIP; include/qengine_cpu.hpp:102-108).
 *  - Gate calls are asynchronous and may be queued for fusion; every value-returning call behaves as if
 *    b200sv_finish() ran first (reference include/qengine_cuda.hpp:167-181).
 *  - An instance is not thread-safe; distinct instances may be driven from distinct host threads
 *    (QPager does, reference src/qpager.cpp:423).
 */
#ifndef B200SV_H
#define B200SV_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200SV_OK 0
#define B200SV_EINVAL (-1) /* bad argument (adapter: std::invalid_argument) */
#define B200SV_ENOMEM (-2) /* device allocation failed (adapter: Qrack::bad_alloc) */
#define B200SV_ECUDA (-3)  /* CUDA runtime / launch error (adapter: std::runtime_error) */
#define B200SV_ESTATE (-4) /* operation not valid in this state */

typedef struct b200sv_state* b200sv_t;

/* ---- library / device (replaces Qrack::CUDAEngine, reference include/common/cudaengine.cuh:35-243) ---- */
int b200sv_abi_version(void);
const char* b200sv_last_error(void);
int b200sv_device_count(int* count);
/* total/free bytes, SM count, and 1 if `dev` can map `peer`'s memory (NVLink P2P). Any out pointer may be NULL. */
int b200sv_device_info(int dev, uint64_t* total_bytes, uint64_t* free_bytes, int* sm_count);
int b200sv_can_access_peer(int dev, int peer, int* can);

/* ---- lifecycle (QEngineCUDA ctor / dtor / CloneEmpty / Clone / SetDevice; qengine_cuda.hpp:280-330) ---- */
int b200sv_create(int device, int n_qubits, int precision, b200sv_t* out); /* starts as the zero state */
int b200sv_destroy(b200sv_t s);
int b200sv_clone(b200sv_t s, b200sv_t* out);         /* deep copy, same device (QEngine::Clone) */
int b200sv_qubit_count(b200sv_t s, int* n_qubits);
int b200sv_precision(b200sv_t s, int* precision);
int b200sv_device(b200sv_t s, int* device);
int b200sv_set_device(b200sv_t s, int device);       /* migrate (QEngine::SetDevice, qengine.hpp:122-125) */
/* device pointer of the amplitude array (NULL for the zero state) — for zero-copy interop, e.g. torch */
int b200sv_device_ptr(b200sv_t s, void** ptr);
/* adopt an externally owned device buffer of 2^n amplitudes (e.g. a torch tensor); never freed by the library */
int b200sv_create_external(int device, int n_qubits, int precision, void* device_ptr, b200sv_t* out);

/* point an external-buffer state at another caller-owned buffer of the same size (double-buffered exchanges) */
int b200sv_rebind_external(b200sv_t s, void* device_ptr);

/* run this state's work on a caller-owned CUDA stream (e.g. torch's current stream, so that NCCL collectives issued by
 * torch.distributed and the engine's kernels are ordered on one stream and can be timed with one pair of events).
 * `stream` is a cudaStream_t passed as void* (0 = the legacy default stream); adopt == 0 restores a private stream. */
int b200sv_set_stream(b200sv_t s, void* stream, int adopt);

/* ---- state I/O (QEngine page ops, qengine.hpp:127-145; CPU semantics src/qengine/state.cpp:66-351) ---- */
int b200sv_set_permutation(b200sv_t s, uint64_t perm, double phase_re, double phase_im); /* SetPermutation :228-254 */
int b200sv_zero(b200sv_t s);                         /* ZeroAmplitudes: frees the buffer */
int b200sv_is_zero(b200sv_t s, int* is_zero);        /* IsZeroAmplitude */
int b200sv_set_state(b200sv_t s, const void* host_amps);                 /* SetQuantumState :308-319 */
int b200sv_get_state(b200sv_t s, void* host_amps);                       /* GetQuantumState :322-335 */
int b200sv_get_probs(b200sv_t s, void* host_probs);                      /* GetProbs :338-351 */
int b200sv_get_page(b200sv_t s, void* host_amps, uint64_t offset, uint64_t length);       /* :66-79 */
int b200sv_set_page(b200sv_t s, const void* host_amps, uint64_t offset, uint64_t length); /* :80-98 */
/* dst[dst_off .. +len) = src[src_off .. +len): SetAmplitudePage(engine, ...) :99-133 (device->device, P2P if needed) */
int b200sv_copy_page(b200sv_t dst, b200sv_t src, uint64_t src_off, uint64_t dst_off, uint64_t length);
int b200sv_shuffle(b200sv_t a, b200sv_t b);          /* ShuffleBuffers :134-163: swap a[half..] with b[..half] */
int b200sv_copy_state(b200sv_t dst, b200sv_t src);   /* CopyStateVec :165-185 */
int b200sv_get_amplitude(b200sv_t s, uint64_t perm, double* re, double* im);              /* :187-201 */
int b200sv_set_amplitude(b200sv_t s, uint64_t perm, double re, double im);                /* :203-226 */

/* ---- gates ---- */
/* QEngine::Apply2x2 (qengine.hpp:281-282; CPU src/qengine/state.cpp:392-533).  For every base index i
 * with zero bits inserted at each powers_sorted[k]: (a,b) = (psi[i+off1], psi[i+off2]);
 * psi[i+off1] = nrm*(m0*a + m1*b); psi[i+off2] = nrm*(m2*a + m3*b).  m8 = {m0.re,m0.im,...,m3.im}.
 * If norm_out != NULL the call also returns sum |psi'|^2 over the touched amplitudes, with amplitudes
 * whose |.|^2 < norm_thresh set to zero and excluded (NORM_THRESH_KERNEL :361-382); this forces a flush. */
int b200sv_apply2x2(b200sv_t s, uint64_t off1, uint64_t off2, const double* m8, int bit_count,
    const uint64_t* powers_sorted, double nrm, double norm_thresh, double* norm_out);
/* XMask (state.cpp:965-1007), PhaseParity (:1009-1054), PhaseRootNMask (:1056-1092) */
int b200sv_xmask(b200sv_t s, uint64_t mask);
int b200sv_phase_parity(b200sv_t s, double radians, uint64_t mask);
int b200sv_phase_root_n_mask(b200sv_t s, int n, uint64_t mask);
/* UniformParityRZ / CUniformParityRZ (state.cpp:1200-1264): control_mask==0 -> uncontrolled */
int b200sv_uniform_parity_rz(b200sv_t s, uint64_t control_mask, uint64_t mask, double angle);
/* UniformlyControlledSingleBit (state.cpp:1094-1198): mtrxs = a table of 2^(n_controls + n_skip) matrices of 8 doubles.  The
 * control bits of a pair's base index (controls[j] -> bit j) get a zero bit inserted at each skip power, in the order given,
 * and skip_value_mask ORed in; that entry is applied, times nrm.  B200SV_EINVAL unless n_controls + n_skip <= 30, controls
 * (when n_controls > 0), skip_powers (when n_skip > 0) and mtrxs are non-NULL, every skip power is a power of two below
 * 2^(n_controls + n_skip), and skip_value_mask is below 2^(n_controls + n_skip). */
int b200sv_uniformly_controlled(b200sv_t s, int n_controls, const int* controls, int target, const double* mtrxs,
    int n_skip, const uint64_t* skip_powers, uint64_t skip_value_mask, double nrm);
/* ApplyM (qengine.hpp:161-166; state.cpp:2167-2196): psi[i] = ((i&mask)==result) ? nrm*psi[i] : 0 */
int b200sv_apply_m(b200sv_t s, uint64_t mask, uint64_t result, double nrm_re, double nrm_im);
/* ForceMParity collapse part (state.cpp:2052-2107): keep parity==result, zero the rest; returns kept norm */
int b200sv_collapse_parity(b200sv_t s, uint64_t mask, int result, double* kept_norm);

/* ---- reductions (state.cpp:1751-1993, 2109-2268) ---- */
/* sum |psi[i]|^2 over i with (i & mask) == perm : Prob (mask=perm=2^q), ProbReg, ProbMask */
int b200sv_prob_mask(b200sv_t s, uint64_t mask, uint64_t perm, double* out);
int b200sv_prob_parity(b200sv_t s, uint64_t mask, double* out);
/* probs[k] for every permutation k of the bits in `mask` (ProbMaskAll, qinterface.cpp:423-476); host_probs has
 * 2^popcount(mask) entries of the state's real type */
int b200sv_prob_mask_all(b200sv_t s, uint64_t mask, void* host_probs);
/* sum |psi|^2 with |.|^2 >= thresh (UpdateRunningNorm / par_norm, parallel_for.cpp:244-300) */
int b200sv_norm(b200sv_t s, double norm_thresh, double* out);
/* psi *= polar(1/sqrt(nrm), phase_arg) with floor-zeroing below norm_thresh (NormalizeState :2198-2248) */
int b200sv_normalize(b200sv_t s, double nrm, double norm_thresh, double phase_arg);
/* <a|b> (SumSqrDiff :2109-2165) */
int b200sv_inner(b200sv_t a, b200sv_t b, double* re, double* im);
/* sum_i |psi[i]|^2 * ((i >> start) & (2^length - 1))  (GetExpectation, utility.cpp); the moments sweep below with
 * perms (0, 2^p) on qubit start + p */
int b200sv_expectation(b200sv_t s, int start, int length, double* out);

/* ---- observables: one read-only sweep each instead of the 2^n ProbAll(i) calls of the QInterface defaults
 * (src/qinterface/qinterface.cpp:478-800).  Queued gates are flushed first; the memoised Prob marginals stay valid and
 * the state is not written.  The zero state returns zeros without a launch.  Every term is accumulated in double.
 *
 * Weighted moments: out[0] = sum_i |psi_i|^2, out[1] = sum_i |psi_i|^2 (w_i - center), out[2] = sum_i |psi_i|^2 (w_i - center)^2,
 * with w_i depending on the bits of i at the k distinct qubits bits[0..k-1]:
 *   bits form   w_i = offset + sum_p perms[2p + bit(i, bits[p])], summed in uint64 (exact) and converted to double once —
 *               the retIndex of ExpectationBitsFactorized / VarianceBitsFactorized (:542-618);
 *   floats form w_i = prod_p weights[2p + bit(i, bits[p])] — ExpectationFloatsFactorized (:771-806) and
 *               VarianceFloatsFactorized (:620-657).
 * k = 0 gives w = offset (bits form) or 1 (floats form).  out[1] with center 0 is the expectation; out[2] with center = that
 * expectation is the true variance (a second sweep, which avoids the cancellation of E[w^2] - E[w]^2).  Note that the
 * reference's VarianceFloatsFactorized for k >= 2 returns the UNSQUARED sum_i p_i (w_i - mean) (:653) = mean (1 - out[0]);
 * its 1-bit branch squares.  B200SV_EINVAL when k < 0, bits / the table / out is NULL where needed, a qubit is outside
 * [0, n) or repeated, or (bits form) offset + sum_p max(perms[2p], perms[2p + 1]) exceeds 2^64 - 1. */
int b200sv_moments_bits(b200sv_t s, int k, const int* bits, const uint64_t* perms, uint64_t offset, double center,
    double* out);
int b200sv_moments_floats(b200sv_t s, int k, const int* bits, const double* weights, double center, double* out);
/* Pauli string P with X on x & ~z, Y on x & z, Z on z & ~x: out[0] = sum |psi|^2, out[1] = <psi|P|psi>
 * = sum_j conj(psi[j ^ x]) i^popcount(x & z) (-1)^popcount(j & z) psi[j], every pair (j, j ^ x) read once.  What
 * ExpectationPauliAll (:715-769) computes by applying H / IS.H basis gates, running the Floats sweep with weights (1, -1)
 * and undoing the gates — here without writing the state.  B200SV_EINVAL when out is NULL or a mask is >= 2^n. */
int b200sv_expectation_pauli(b200sv_t s, uint64_t x_mask, uint64_t z_mask, double* out);
/* Cross-page Pauli term: with phi = the 2^n amplitudes at `partner` (same precision; a device pointer readable from s's device: another
 * state's buffer, s's own buffer, or a peer mapping of another process's page), out[0] + i out[1] = sum_j conj(phi[j ^ x]) (-1)^popcount(j & z) psi[j]
 * and out[2] = sum_j |psi_j|^2, every term in double.  Read-only on both buffers; queued gates of s (and a pending re-page) are flushed first.
 * The zero state returns zeros without a launch.  B200SV_EINVAL when partner or out is NULL or a mask is >= 2^n. */
int b200sv_expectation_pauli_pair(b200sv_t s, const void* partner, uint64_t x_mask, uint64_t z_mask, double* out);
/* Reduced density matrix on the k qubits qubits[0..k-1] (GetReducedDensityMatrix, qinterface.cpp:886-944):
 * out[2 (i 2^k + j)] + i out[2 (i 2^k + j) + 1] = sum_e psi[i, e] conj(psi[j, e]), where bit p of i and j is
 * qubit qubits[p] (the order given, not sorted) and e runs over the other qubits.  Not normalised.
 * Read-only; the zero state gives zeros.  B200SV_EINVAL when k < 0, k > B200SV_RDM_MAX_QUBITS (14), k > n,
 * qubits (k > 0) or out is NULL, a qubit is outside [0, n) or repeated.  B200SV_ENOMEM when the device buffer
 * cannot be had. */
#define B200SV_RDM_MAX_QUBITS 14
int b200sv_reduced_density_matrix(b200sv_t s, int k, const int* qubits, double* out);
/* Weighted moments in a per-qubit basis (ExpVarUnitaryAll, qinterface.cpp:478-540): with A_p the 2x2 matrix mats8[8p .. 8p + 7]
 * (m00, m01, m10, m11, each re, im) on qubit bits[p], phi = (A_0 (x) .. (x) A_{k-1} on those qubits) psi, and
 * out = the three moments of b200sv_moments_floats above computed on phi instead of psi: out[0] = sum |phi_i|^2,
 * out[1] = sum |phi_i|^2 (w_i - center), out[2] = sum |phi_i|^2 (w_i - center)^2, w_i = prod_p weights[2p + bit(i, bits[p])].
 * What the reference gets by applying A_p (the inverse of the caller's basis matrix, or U(-theta, -phi, -lambda)) to every
 * listed qubit, running the Floats query and applying the gates again — here without writing the state.  Queued gates are
 * flushed; the state and the memoised Prob marginals are kept; the zero state returns zeros without a launch.
 * B200SV_EINVAL when k < 1, k > B200SV_BASIS_MAX_QUBITS (12), bits / mats8 / weights / out is NULL, or a qubit is outside
 * [0, n) or repeated. */
#define B200SV_BASIS_MAX_QUBITS 12
int b200sv_moments_basis(b200sv_t s, int k, const int* bits, const double* mats8, const double* weights, double center,
    double* out);
/* index of the largest |psi|^2 (HighestProbAll :1995-2024) */
int b200sv_highest_prob(b200sv_t s, uint64_t* perm);
/* The n most probable basis states (HighestProbAll(n), qinterface.cpp:962-1003): perms_out[0..n) sorted by
 * P(i) = min(|psi_i|^2, 1) descending, then by index ascending, P computed in double (fp32: (double)re^2 + (double)im^2).
 * Indices with P = 0 are never listed; when fewer than n have P > 0 the list ends with zeros.  Exact: the reference's early
 * exit on its running sum is not reproduced.  Read-only; the zero state gives n zeros.  n = 0 does nothing.  B200SV_EINVAL
 * when perms_out is NULL (n > 0) or n > 2^qubits; B200SV_ENOMEM when the device buffer (16 B per listed state, beyond 1 MiB)
 * cannot be had. */
int b200sv_highest_probs(b200sv_t s, uint64_t n, uint64_t* perms_out);
/* The n best basis states of HighestProbAll(n) under a caller's tie key t(i) = key_xor ^ (OR over the bits b set in i of
 * 2^key_pos[b]), key_pos[0..qubits): keys_out[t] = t(i) of the t-th entry and probs_out[t] = its P = min(|psi_i|^2, 1) in
 * double (fp32: (double)re^2 + (double)im^2), both zero-filled past the last P > 0.  Sorted by P descending, then t(i)
 * ascending.  key_pos == NULL means key_pos[b] = b; with key_xor = 0 that is the order of b200sv_highest_probs.  A page of a
 * sharded state passes its logical qubits as key_pos and its rank's logical bits (and pending inversions) as key_xor, so that
 * its ties go to the smaller logical index.  Read-only; queued gates are flushed first; the zero state gives zeros.  n = 0
 * does nothing once the key is checked.  B200SV_EINVAL: keys_out or probs_out NULL with n > 0; n > 2^qubits; key_bits outside
 * [qubits, 64]; a key position negative, repeated or >= key_bits; key_xor >= 2^key_bits.  B200SV_ENOMEM as
 * b200sv_highest_probs. */
int b200sv_highest_probs_keyed(b200sv_t s, uint64_t n, int key_bits, const int* key_pos, uint64_t key_xor,
    uint64_t* keys_out, double* probs_out);
/* LossySaveStateVector (reference include/statevector_turboquant.hpp; QEngineCUDA cuda.cu:3017-3035): writes the TurboQuant
 * file of the current state to `path`, block power p (1..6), `bits` per coordinate (1..16), every block rotated by the
 * rotation of `seed`.  Bit-exact with the reference codec in plain sequential IEEE arithmetic.  Read-only: queued gates are
 * flushed, the state and the memoised marginals are kept.  The zero state is encoded without a launch.  B200SV_EINVAL for a
 * NULL path, p or bits out of range, or a file that cannot be written. */
int b200sv_lossy_save(b200sv_t s, const char* path, int p, int bits, uint64_t seed);
/* header + record geometry of a file for a state of `precision` (32 / 64): its qubit count (the adapter resizes before
 * loading), block power and bits.  B200SV_EINVAL when the file cannot be opened, its capacity is not a power of two,
 * num_blocks does not match, or the first record's D or NWORDS does not (a file of the other precision). */
int b200sv_lossy_probe(const char* path, int precision, int* n_qubits, int* p, int* bits);
/* LossyLoadStateVector: decodes the file into s, whose qubit count must equal the file's.  One rotation is built per distinct
 * seed.  B200SV_EINVAL (state untouched) for a file that cannot be opened, a qubit count that differs, p outside 1..6, a
 * block whose D is not BLOCK, BITS differing between blocks or outside 1..16, NWORDS not (2 D BITS + 63) / 64, a capacity
 * that is not a power of two, or a length that does not match the state's precision; a malformed record found after the
 * first chunk of 64 MiB of staging has been decoded leaves the zero state. */
int b200sv_lossy_load(b200sv_t s, const char* path);
/* TEST HOOK (host only): the dim x dim column-major rotation of `seed` in the given precision (32: float, 64: double) */
int b200sv_lossy_rotation(int dim, int precision, uint64_t seed, void* out);
/* smallest index i with |psi[i]|^2 > REAL1_EPSILON and cumulative cum = sum_{j<=i} |psi[j]|^2 > rnd or 1 - cum <= FP_NORM_EPSILON,
 * else the last index with |psi|^2 > REAL1_EPSILON, else 2^n - 1 (MAll :2026-2050) */
int b200sv_sample(b200sv_t s, double rnd, uint64_t* perm);
/* n_shots samples of the whole register WITHOUT collapse in one call (MultiShotMeasureMask, src/qengine/qengine.cpp:542-609:
 * the k measured bits are read off each sampled basis state — same distribution as drawing from the 2^k histogram);
 * rnds[i] in [0,1) -> perms[i] = b200sv_sample(s, rnds[i]) (MAll's search, its FP_NORM_EPSILON early exit included). */
int b200sv_sample_many(b200sv_t s, int n_shots, const double* rnds, uint64_t* perms);
/* The samples of b200sv_sample_many mapped through a caller's tie key t(i) = key_xor ^ (OR over the bits b set in i of
 * 2^key_pos[b]), key_pos[0..qubits): keys_out[i] = t(b200sv_sample(s, rnds[i])).  key_pos == NULL means key_pos[b] = b.  A page
 * of a sharded state passes its logical qubits and its rank's logical bits (and pending inversions), so its samples come back
 * as logical indices.  Read-only; queued gates are flushed first.  The zero state gives t(2^n - 1) for every shot without a
 * launch; any other state costs two launches (chunk sums, search) whatever n_shots is.  B200SV_EINVAL: n_shots < 0; rnds or
 * keys_out NULL with n_shots > 0; the key as in b200sv_highest_probs_keyed (key_bits outside [qubits, 64]; a key position
 * negative, repeated or >= key_bits; key_xor >= 2^key_bits). */
int b200sv_sample_keyed(b200sv_t s, int n_shots, const double* rnds, int key_bits, const int* key_pos, uint64_t key_xor,
    uint64_t* keys_out);

/* ---- structure (state.cpp:1271-1748; utility.cpp:54-68) ---- */
/* a <- a (x) b with b's qubits inserted at `start` (Compose :1368-1459; start==n_a is the append form :1271-1362) */
int b200sv_compose(b200sv_t a, b200sv_t b, int start);
/* DecomposeDispose (:1551-1696): remove qubits [start,start+length); dest (may be NULL = Dispose) receives them */
int b200sv_decompose(b200sv_t s, int start, int length, b200sv_t dest);
/* Dispose(start,length,perm) (:1708-1748): pure gather of the slice where the disposed bits == perm */
int b200sv_dispose_perm(b200sv_t s, int start, int length, uint64_t perm);

/* ---- multi-process exchange over NVLink peer memory (one process per GPU; SURVEY.md §8e) ----
 * Pages are plain cudaMalloc allocations so that they can be exported with CUDA IPC and mapped by the peer processes.
 * b200sv_exchange_scatter is the fused "re-page" step: ONE kernel reads this rank's page once and stores every 16-byte
 * chunk straight into the destination rank's page through the peer mapping (the element with local index i goes to
 * rank r' = the bits of i at victim_bits[0..k-1], to index i with those bits replaced by this rank's bits) — i.e. the
 * k rank-index qubits are exchanged with k arbitrary local qubits without any local pre-permutation sweep and without
 * staging (reference: QPager re-pages with SetAmplitudePage / 2x ShuffleBuffers, src/qpager.cpp:316-367,425-432).
 * 1 <= k <= 8 and 0 <= rank < 2^k, else B200SV_EINVAL, as for b200sv_exchange_pull. */
int b200sv_alloc_page(int device, uint64_t bytes, void** ptr);
int b200sv_free_page(int device, void* ptr);
int b200sv_ipc_export(int device, void* ptr, unsigned char handle_out[64]);
int b200sv_ipc_import(int device, const unsigned char handle[64], void** ptr);
int b200sv_ipc_release(int device, void* ptr);
int b200sv_exchange_scatter(b200sv_t s, int k, const int* victim_bits, int rank, void* const* dst_pages);
/* The same re-page in PULL mode, fused into the next gate sweep: declares that this state's content is now the exchanged view
 * of the ranks' current pages (src_pages[r] = rank r's page as mapped in this process, src_pages[rank] = this state's own
 * page; element i of the new page = element (i with the victim bits := this rank's bits) of the page of rank r' = the victim
 * bits of i) and that it lives in out_page from now on.  Nothing is copied by this call: the FIRST fused sweep of the next
 * flush reads its tiles straight through the peer mappings and writes out_page (k_fused_sweep<PULL>), so the exchange costs
 * no pass of its own; a flush with no sweep to carry it runs a plain gather kernel.  The caller orders the ranks: a barrier
 * between the last write of every source page and this call's first use, and none of the source pages may be written until
 * every rank has flushed (the next barrier).  1 <= k <= 3.  (Reference: QPager::MetaSwap / SeparateEngines re-paging,
 * src/qpager.cpp:316-367,425-432, always a separate pass there.) */
int b200sv_exchange_pull(b200sv_t s, int k, const int* victim_bits, int rank, void* const* src_pages, void* out_page);

/* ---- queue / fusion control ---- */
int b200sv_flush(b200sv_t s);  /* launch everything queued; does not wait */
int b200sv_finish(b200sv_t s); /* flush + wait for the device (QInterface::Finish) */
/* mode 0: every gate is its own launch (reference-like); 1: fused multi-gate sweeps (default) */
int b200sv_set_fusion(b200sv_t s, int mode);

/* ---- QAlu family (SURVEY.md §8f N3): basis-state maps, one out-of-place sweep each -------------------------------
 * Replaces the QEngineCPU members of src/qengine/arithmetic.cpp that a QEngine must provide (include/qalu.hpp:34-236,
 * include/qengine.hpp ROL).  bitCapIntOcl arguments travel as uint64_t; `ctrl_mask` = OR of 2^control (0: uncontrolled).
 * Pre-steps the reference performs at QInterface level (SetReg of the carry register, M/X of the carry qubit) are the
 * adapter's job, as in the reference.  A zero (unallocated) state is left untouched (CHECK_ZERO_SKIP). */
int b200sv_rol(b200sv_t s, int shift, int start, int length);                              /* arithmetic.cpp:23-70 */
int b200sv_inc(b200sv_t s, uint64_t to_add, int start, int length, uint64_t ctrl_mask);    /* INC :73-118, CINC :121-172 */
int b200sv_incdecc(b200sv_t s, uint64_t to_mod, int start, int length, int carry_index);   /* :175-224 */
int b200sv_incs(b200sv_t s, uint64_t to_add, int start, int length, int overflow_index);   /* :227-309 */
/* overflow_index < 0: the carry-only form (:312-361); else overflow flag + carry (:364-419) */
int b200sv_incdecsc(b200sv_t s, uint64_t to_mod, int start, int length, int overflow_index, int carry_index);
/* inverse = 0: MUL / CMUL (:422-471, :488-573); 1: DIV / CDIV */
int b200sv_muldiv(b200sv_t s, int inverse, uint64_t to_mul, int start, int carry_start, int length, uint64_t ctrl_mask);
/* kind 0: MULModNOut, 1: IMULModNOut, 2: POWModNOut and their controlled forms (:595-775) */
int b200sv_modnout(b200sv_t s, int kind, uint64_t to_mod, uint64_t mod_n, int in_start, int out_start, int length,
    uint64_t ctrl_mask);
/* kind 0: IndexedLDA (:983-1083), 1: IndexedADC (:1086-1260), 2: IndexedSBC (:1263-1444); `values` is a HOST table of
 * 2^index_length entries of (value_length+7)/8 bytes; carry_in = the classical carry the adapter measured */
int b200sv_indexed(b200sv_t s, int kind, int index_start, int index_length, int value_start, int value_length,
    int carry_index, int carry_in, const unsigned char* values);
int b200sv_hash(b200sv_t s, int start, int length, const unsigned char* values);           /* :1447-1506 */
/* flag_index < 0: PhaseFlipIfLess (:1703-1720); else CPhaseFlipIfLess (:1678-1701) */
int b200sv_phase_flip_if_less(b200sv_t s, uint64_t greater_perm, int start, int length, int flag_index);

/* Batched submission (SURVEY 8f N4; what the reference does gate by gate in QCircuit::Run, include/qcircuit.hpp:121-324,
 * src/qcircuit.cpp:173-281): n_gates single-target Apply2x2 calls in ONE ABI call.  Gate i is Apply2x2(off1[i], off2[i],
 * mats8 + 8 i, powers = the bits of pmasks[i], nrm = 1, no norm output); off1[i] ^ off2[i] must be a single power.  Identical
 * in effect to n_gates b200sv_apply2x2 calls (same queue, same fused planner), without the per-gate host round trip. */
int b200sv_apply_gates(b200sv_t s, int n_gates, const uint64_t* off1, const uint64_t* off2, const uint64_t* pmasks,
    const double* mats8);

/* Test hook (no device needed, never on the engine's path): plan + encode the gate list exactly as b200sv_apply2x2 /
 * the fused flush would, then interpret every encoded sweep program on a HOST state vector (n_qubits <= 30;
 * interleaved re/im of the given precision).  Gate i is Apply2x2(off1[i], off2[i], mats8 + 8 i, powers = bits of
 * pmasks[i]) in its single-target form.  `pytest -m "not gpu"` checks scheduler + encoder against the oracle with it. */
int b200sv_emulate_fused(int n_qubits, int precision, int n_gates, const uint64_t* off1, const uint64_t* off2,
    const uint64_t* pmasks, const double* mats8, void* host_state);
/* DIAGNOSTIC (host only): what one flush of this gate list would launch — fused sweeps, register passes, device ops
 * (scripts/shard_sweep_count.py counts the sweeps of a sharded step with it) */
int b200sv_plan_gates(int n_qubits, int precision, int n_gates, const uint64_t* off1, const uint64_t* off2,
    const uint64_t* pmasks, const double* mats8, int* n_sweeps, int* n_passes, int* n_ops);
/* TEST HOOK (host only): b200sv_emulate_fused with a pending b200sv_exchange_pull — src_states[r] are HOST arrays standing in
 * for the ranks' pages, out_state receives this rank's new page after the gates (first sweep reads through the pull mapping). */
int b200sv_emulate_fused_pull(int n_qubits, int precision, int n_gates, const uint64_t* off1, const uint64_t* off2,
    const uint64_t* pmasks, const double* mats8, int k, const int* victim_bits, int rank, void* const* src_states,
    void* out_state);

typedef struct b200sv_stats {
    uint64_t gates_submitted;  /* apply2x2-class calls accepted */
    uint64_t kernel_launches;  /* CUDA kernels launched by this state */
    uint64_t fused_sweeps;     /* fused-window launches */
    uint64_t fused_gates;      /* gates executed inside fused sweeps */
    uint64_t single_launches;  /* unfused single-gate launches */
    uint64_t bytes_swept;      /* physical bytes read+written by gate kernels */
    uint64_t pull_sweeps;      /* fused sweeps that also carried a pending re-page (b200sv_exchange_pull) */
} b200sv_stats;
int b200sv_get_stats(b200sv_t s, b200sv_stats* out);
int b200sv_reset_stats(b200sv_t s);

/* CUDA-event timing of the gate stream: begin records an event on the state's stream, end records another,
 * waits, and returns the elapsed milliseconds (used by bench.py: torch.cuda.Event only sees torch's stream). */
int b200sv_timer_begin(b200sv_t s);
int b200sv_timer_end(b200sv_t s, double* elapsed_ms);
/* write `bytes` of a scratch buffer on the state's device/stream (L2 flush between timed iterations) */
int b200sv_flush_l2(b200sv_t s, uint64_t bytes);

#ifdef __cplusplus
}
#endif
#endif /* B200SV_H */
