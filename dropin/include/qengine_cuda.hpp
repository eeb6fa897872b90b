// qengine_cuda.hpp — drop-in replacement of the reference header of the same name
// (reference include/qengine_cuda.hpp) : class Qrack::QEngineCUDA on the H100 state-vector core.
//
// The class keeps the reference's name, base class and shared positional constructor signature
// (reference include/qengine_cuda.hpp:280-284) so that include/qfactory.hpp:80,128,172,237, QPager, QHybrid, QUnit,
// QUnitMulti, the unit tests and the benchmarks compile and run UNCHANGED with ENABLE_CUDA=1.  It contains no CUDA
// code: every sweep over amplitudes is one call into the C ABI of include/b200sv.h (libb200sv.so, hand-written
// sm_90a kernels).  What stays here is QEngine-level bookkeeping only: runningNorm / doNormalize, argument checks that
// must throw std::invalid_argument, and the zero-state shortcuts.
#pragma once

#include "common/cudaengine.cuh"
#include "qengine.hpp"

struct b200sv_state;

namespace Qrack {

class QEngineCUDA;
typedef std::shared_ptr<QEngineCUDA> QEngineCUDAPtr;

class QEngineCUDA : public QEngine {
protected:
    b200sv_state* sv;
    int64_t deviceID;
    bool svCountSynced; // guards SetQubitCount() against re-creating the handle after a structural ABI call

    void Check(int rc) const;
    void ResizeZero(bitLenInt qb);
    void SyncQubitCount();
    QEngineCUDAPtr Cast(QInterfacePtr p, const char* what) const;

    /// QInterface::TryDecompose (src/qinterface/qinterface.cpp:836-853) adopts another instance's state through this
    /// protected hook; the reference engines share the buffer (include/qengine_cpu.hpp:47-55), here it is a device copy.
    using QEngine::Copy;
    void Copy(QInterfacePtr orig) { Copy(std::dynamic_pointer_cast<QEngineCUDA>(orig)); }
    void Copy(QEngineCUDAPtr orig);

    /// OR of 2^control; throws std::invalid_argument like ThrowIfQbIdArrayIsBad (common/qrack_functions.hpp)
    uint64_t CtrlMask(const std::vector<bitLenInt>& controls, const char* what) const;

    /// the sum-form weights as uint64 (false: a perm, the offset or the largest weight does not fit — the base class loops)
    bool BitsWeights(const std::vector<bitLenInt>& bits, const std::vector<bitCapInt>& perms, const bitCapInt& offset,
        std::vector<int>& b, std::vector<uint64_t>& p, uint64_t& off) const;
    /// (S0, S1, S2) of b200sv_moments_bits / _floats after the doNormalize step
    void Moments(const std::vector<int>& b, const std::vector<uint64_t>& p, uint64_t off, double center, double* out);
    void MomentsFloats(const std::vector<bitLenInt>& bits, const std::vector<real1_f>& weights, double* out);
    /// drops PauliI as the reference's loop does (some survive it and count as PauliZ); false when a qubit is out of bounds or
    /// repeated (the base class then throws what it throws)
    bool PauliMasks(std::vector<bitLenInt>& bits, const std::vector<Pauli>& paulis, uint64_t& x, uint64_t& z) const;
    /// the Floats query of ExpVarUnitaryAll on the state with mats[4p .. 4p + 3] applied to bits[p], read-only
    real1_f BasisMoments(bool isExp, const std::vector<bitLenInt>& bits, const complex* mats, std::vector<real1_f> eigenVals);

    // ExpVarUnitaryAll (qinterface.cpp:478-540) applies a basis gate to every listed qubit, runs the Floats query and applies
    // the gates again: five state passes.  Here the query is one read-only sweep over the transformed blocks
    // (b200sv_moments_basis).  The matrix form leaves the state untouched.  The U3 form then applies U(theta, phi, lambda)
    // U(-theta, -phi, -lambda) as one gate per qubit: the reference's undo is not the inverse of its first gate, and this keeps
    // its post-state.  More than B200SV_BASIS_MAX_QUBITS qubits go to the base class.
    real1_f ExpVarUnitaryAll(bool isExp, const std::vector<bitLenInt>& bits, const std::vector<std::shared_ptr<complex>>& basisOps,
        std::vector<real1_f> eigenVals = {}) override;
    real1_f ExpVarUnitaryAll(bool isExp, const std::vector<bitLenInt>& bits, const std::vector<real1_f>& basisOps,
        std::vector<real1_f> eigenVals = {}) override;

public:
    /// 1 / OclMemDenom of device memory is the most a single state vector should take (test/benchmarks_main.cpp:288)
    static const bitCapIntOcl OclMemDenom = 3U;

    QEngineCUDA(bitLenInt qBitCount, const bitCapInt& initState, qrack_rand_gen_ptr rgp = nullptr,
        const complex& phaseFac = CMPLX_DEFAULT_ARG, bool doNorm = false, bool randomGlobalPhase = true,
        bool useHostMem = false, int64_t devID = -1, bool useHardwareRNG = true, bool ignored = false,
        real1_f norm_thresh = REAL1_EPSILON, std::vector<int64_t> ignored2 = {}, bitLenInt ignored4 = 0U,
        real1_f ignored3 = _qrack_qunit_sep_thresh);
    ~QEngineCUDA();

    bool isOpenCL() override { return true; }
    void SetDevice(int64_t dID) override;
    int64_t GetDevice() override { return deviceID; }
    bitCapIntOcl GetMaxSize();
    b200sv_state* Handle() { return sv; }

    void SetQubitCount(bitLenInt qb) override;
    void Finish() override;
    bool isFinished() override;
    void Dump() override {}

    // ---- QEngine page / buffer virtuals (qengine.hpp:127-152) ----
    void ZeroAmplitudes() override;
    void CopyStateVec(QEnginePtr src) override;
    bool IsZeroAmplitude() override;
    void GetAmplitudePage(complex* pagePtr, bitCapIntOcl offset, bitCapIntOcl length) override;
    void SetAmplitudePage(const complex* pagePtr, bitCapIntOcl offset, bitCapIntOcl length) override;
    void SetAmplitudePage(QEnginePtr pageEnginePtr, bitCapIntOcl srcOffset, bitCapIntOcl dstOffset, bitCapIntOcl length) override;
    void ShuffleBuffers(QEnginePtr engine) override;
    QEnginePtr CloneEmpty() override;
    QInterfacePtr Clone() override;
    void QueueSetDoNormalize(bool doNorm) override { doNormalize = doNorm; }
    void QueueSetRunningNorm(real1_f runningNrm) override { runningNorm = (real1)runningNrm; }

    // ---- state access (qinterface.hpp:313-344) ----
    void SetQuantumState(const complex* inputState) override;
    void GetQuantumState(complex* outputState) override;
    void GetProbs(real1* outputProbs) override;
    complex GetAmplitude(const bitCapInt& perm) override;
    void SetAmplitude(const bitCapInt& perm, const complex& amp) override;
    void SetPermutation(const bitCapInt& perm, const complex& phaseFac = CMPLX_DEFAULT_ARG) override;

    // ---- the gate hot path ----
    void Apply2x2(bitCapInt offset1, bitCapInt offset2, const complex* mtrx, bitLenInt bitCount, bitCapInt const* qPowersSorted,
        bool doCalcNorm, real1_f norm_thresh = REAL1_DEFAULT_ARG);
    using QEngine::ApplyM;
    void ApplyM(const bitCapInt& regMask, const bitCapInt& result, const complex& nrm) override;
    void XMask(const bitCapInt& mask) override;
    void PhaseParity(real1_f radians, const bitCapInt& mask) override;
    void PhaseRootNMask(bitLenInt n, const bitCapInt& mask) override;
    using QEngine::UniformlyControlledSingleBit;
    void UniformlyControlledSingleBit(const std::vector<bitLenInt>& controls, bitLenInt qubitIndex, const complex* mtrxs,
        const std::vector<bitCapInt>& mtrxSkipPowers, const bitCapInt& mtrxSkipValueMask);
    void UniformParityRZ(const bitCapInt& mask, real1_f angle) override;
    void CUniformParityRZ(const std::vector<bitLenInt>& controls, const bitCapInt& mask, real1_f angle) override;

    // ---- probabilities / measurement ----
    real1_f Prob(bitLenInt qubit) override;
    real1_f CtrlOrAntiProb(bool controlState, bitLenInt control, bitLenInt target) override;
    real1_f ProbReg(bitLenInt start, bitLenInt length, const bitCapInt& permutation) override;
    real1_f ProbMask(const bitCapInt& mask, const bitCapInt& permutation) override;
    void ProbMaskAll(const bitCapInt& mask, real1* probsArray) override;
    void ProbRegAll(bitLenInt start, bitLenInt length, real1* probsArray) override;
    // SURVEY 8f N1: the QInterface default walks all 2^n basis states on the host (src/qinterface/qinterface.cpp:446-476)
    void ProbBitsAll(const std::vector<bitLenInt>& bits, real1* probsArray) override;
    // QEngine's versions (src/qengine/qengine.cpp:542-609) build the 2^k histogram first; with many measured qubits the
    // shots are sampled as basis states on the device instead (b200sv_sample_many) — same distribution
    std::map<bitCapInt, int> MultiShotMeasureMask(const std::vector<bitCapInt>& qPowers, unsigned shots) override;
    void MultiShotMeasureMask(const std::vector<bitCapInt>& qPowers, unsigned shots, unsigned long long* shotsArray) override;
    real1_f ProbParity(const bitCapInt& mask) override;
    bool ForceMParity(const bitCapInt& mask, bool result, bool doForce = true) override;
    bitCapInt MAll() override;
    bitCapInt HighestProbAll(); // device arg-max; the QInterface default asks ProbAll() for every permutation
    // top n as a device radix select (the default asks ProbAll() for every permutation and keeps the best n by insertion);
    // exact, without the default's early exit on its running sum.  n > maxQPower throws before anything is launched.
    std::vector<bitCapInt> HighestProbAll(size_t n) override;
    // lossy checkpoints (the TurboQuant file of statevector_turboquant.hpp) encoded / decoded on the device for 1 <= p <= 6 and
    // 1 <= b <= 16; other p or b go to the QInterface default.  An unreadable file zeroes the state, as QEngineCPU does.
    void LossySaveStateVector(std::string f, int p = 6, int b = 4) override;
    void LossyLoadStateVector(std::string f) override;
    real1_f FirstNonzeroPhase() override { return IsZeroAmplitude() ? ZERO_R1_F : QInterface::FirstNonzeroPhase(); }
    real1_f GetExpectation(bitLenInt valueStart, bitLenInt valueLength) override;
    // The QInterface defaults ask ProbAll(i) — one device round trip — for every basis state (qinterface.cpp:478-800); here a
    // k >= 2 query is one read-only sweep (two for VarianceBitsFactorized).  ExpectationBitsAll / VarianceBitsAll and the
    // *Rdm forms reach these through QInterface's own virtual calls; the *UnitaryAll forms reach ExpVarUnitaryAll above.
    real1_f ExpectationBitsFactorized(
        const std::vector<bitLenInt>& bits, const std::vector<bitCapInt>& perms, const bitCapInt& offset = ZERO_BCI) override;
    real1_f VarianceBitsFactorized(
        const std::vector<bitLenInt>& bits, const std::vector<bitCapInt>& perms, const bitCapInt& offset = ZERO_BCI) override;
    real1_f ExpectationFloatsFactorized(const std::vector<bitLenInt>& bits, const std::vector<real1_f>& weights) override;
    real1_f VarianceFloatsFactorized(const std::vector<bitLenInt>& bits, const std::vector<real1_f>& weights) override;
    real1_f ExpectationPauliAll(std::vector<bitLenInt> bits, std::vector<Pauli> paulis) override;
    real1_f VariancePauliAll(std::vector<bitLenInt> bits, std::vector<Pauli> paulis) override;
    // The QInterface default asks GetAmplitude 2^n (1 + 2^k) times (qinterface.cpp:886-944); here it is one read-only sweep.
    // An out-of-range or repeated qubit throws std::invalid_argument; k > B200SV_RDM_MAX_QUBITS goes to the base class.
    void GetReducedDensityMatrix(const std::vector<bitLenInt>& qubits, complex* outputState) override;

    // ---- structure ----
    using QEngine::Compose;
    bitLenInt Compose(QEngineCUDAPtr toCopy);
    bitLenInt Compose(QInterfacePtr toCopy) override { return Compose(Cast(toCopy, "Compose")); }
    bitLenInt Compose(QEngineCUDAPtr toCopy, bitLenInt start);
    bitLenInt Compose(QInterfacePtr toCopy, bitLenInt start) override { return Compose(Cast(toCopy, "Compose"), start); }
    using QEngine::Decompose;
    void Decompose(bitLenInt start, QInterfacePtr dest) override;
    void Dispose(bitLenInt start, bitLenInt length) override;
    void Dispose(bitLenInt start, bitLenInt length, const bitCapInt& disposedPerm) override;
    using QEngine::Allocate;
    bitLenInt Allocate(bitLenInt start, bitLenInt length) override;

    // ---- norm ----
    real1_f SumSqrDiff(QInterfacePtr toCompare) override;
    void NormalizeState(
        real1_f nrm = REAL1_DEFAULT_ARG, real1_f norm_thresh = REAL1_DEFAULT_ARG, real1_f phaseArg = ZERO_R1_F);
    void UpdateRunningNorm(real1_f norm_thresh = REAL1_DEFAULT_ARG) override;

    void ROL(bitLenInt shift, bitLenInt start, bitLenInt length) override;
    void ROR(bitLenInt shift, bitLenInt start, bitLenInt length) override;

#if ENABLE_ALU
    // ---- QAlu (include/qalu.hpp): one device sweep each (include/b200sv.h "QAlu family") ----
    void INC(const bitCapInt& toAdd, bitLenInt start, bitLenInt length) override;
    void CINC(const bitCapInt& toAdd, bitLenInt start, bitLenInt length, const std::vector<bitLenInt>& controls) override;
    void INCDECC(const bitCapInt& toMod, bitLenInt start, bitLenInt length, bitLenInt carryIndex) override;
    void INCS(const bitCapInt& toAdd, bitLenInt start, bitLenInt length, bitLenInt overflowIndex) override;
    void MULModNOut(const bitCapInt& toMod, const bitCapInt& modN, bitLenInt inStart, bitLenInt outStart, bitLenInt length) override;
    void IMULModNOut(const bitCapInt& toMod, const bitCapInt& modN, bitLenInt inStart, bitLenInt outStart, bitLenInt length) override;
    void CMULModNOut(const bitCapInt& toMod, const bitCapInt& modN, bitLenInt inStart, bitLenInt outStart, bitLenInt length,
        const std::vector<bitLenInt>& controls);
    void CIMULModNOut(const bitCapInt& toMod, const bitCapInt& modN, bitLenInt inStart, bitLenInt outStart, bitLenInt length,
        const std::vector<bitLenInt>& controls);
    void PhaseFlipIfLess(const bitCapInt& greaterPerm, bitLenInt start, bitLenInt length) override;
    void CPhaseFlipIfLess(const bitCapInt& greaterPerm, bitLenInt start, bitLenInt length, bitLenInt flagIndex) override;
    void INCDECSC(const bitCapInt& toMod, bitLenInt start, bitLenInt length, bitLenInt carryIndex) override;
    void INCDECSC(const bitCapInt& toMod, bitLenInt start, bitLenInt length, bitLenInt overflowIndex, bitLenInt carryIndex) override;
    void MUL(const bitCapInt& toMul, bitLenInt start, bitLenInt carryStart, bitLenInt length) override;
    void DIV(const bitCapInt& toDiv, bitLenInt start, bitLenInt carryStart, bitLenInt length) override;
    void POWModNOut(const bitCapInt& base, const bitCapInt& modN, bitLenInt inStart, bitLenInt outStart, bitLenInt length) override;
    void CMUL(const bitCapInt& toMul, bitLenInt start, bitLenInt carryStart, bitLenInt length,
        const std::vector<bitLenInt>& controls);
    void CDIV(const bitCapInt& toDiv, bitLenInt start, bitLenInt carryStart, bitLenInt length,
        const std::vector<bitLenInt>& controls);
    void CPOWModNOut(const bitCapInt& base, const bitCapInt& modN, bitLenInt inStart, bitLenInt outStart, bitLenInt length,
        const std::vector<bitLenInt>& controls);
    bitCapInt IndexedLDA(bitLenInt indexStart, bitLenInt indexLength, bitLenInt valueStart, bitLenInt valueLength,
        const unsigned char* values, bool resetValue = true);
    bitCapInt IndexedADC(bitLenInt indexStart, bitLenInt indexLength, bitLenInt valueStart, bitLenInt valueLength,
        bitLenInt carryIndex, const unsigned char* values);
    bitCapInt IndexedSBC(bitLenInt indexStart, bitLenInt indexLength, bitLenInt valueStart, bitLenInt valueLength,
        bitLenInt carryIndex, const unsigned char* values);
    void Hash(bitLenInt start, bitLenInt length, const unsigned char* values) override;
#endif
};

} // namespace Qrack
