// qengine_cuda.cpp — Qrack::QEngineCUDA on the H100 state-vector core (see dropin/include/qengine_cuda.hpp).
//
// Host-side semantics follow QEngineCPU, the parity oracle (reference src/qengine/state.cpp, utility.cpp); every
// method cites the lines it mirrors.  All amplitude work happens behind include/b200sv.h.
#include "qengine_cuda.hpp"

#include "b200sv.h"
#include "qengine_cpu.hpp"
#include "qengine_gpu_util.hpp"

#include <algorithm>
#include <cstring>
#include <fstream>
#include <random>

namespace Qrack {

static const int kPrecision = (int)(8U * sizeof(real1));

void QEngineCUDA::Check(int rc) const
{
    if (rc == B200SV_OK) {
        return;
    }
    const std::string msg = std::string("QEngineCUDA(b200sv): ") + b200sv_last_error();
    if (rc == B200SV_EINVAL) {
        throw std::invalid_argument(msg);
    }
    if (rc == B200SV_ENOMEM) {
        throw bad_alloc(msg);
    }
    throw std::runtime_error(msg);
}

QEngineCUDAPtr QEngineCUDA::Cast(QInterfacePtr p, const char* what) const
{
    QEngineCUDAPtr c = std::dynamic_pointer_cast<QEngineCUDA>(p);
    if (!c) {
        throw std::invalid_argument(std::string("QEngineCUDA::") + what + " argument is not a QEngineCUDA!");
    }
    return c;
}

QEngineCUDA::QEngineCUDA(bitLenInt qBitCount, const bitCapInt& initState, qrack_rand_gen_ptr rgp, const complex& phaseFac,
    bool doNorm, bool randomGlobalPhase, bool useHostMem, int64_t devID, bool useHardwareRNG, bool ignored,
    real1_f norm_thresh, std::vector<int64_t> ignored2, bitLenInt ignored4, real1_f ignored3)
    : QEngine(qBitCount, rgp, doNorm, randomGlobalPhase, useHostMem, useHardwareRNG, norm_thresh)
    , sv(nullptr)
    , deviceID(devID)
    , svCountSynced(false)
{
    if (deviceID < 0) {
        deviceID = (int64_t)CUDAEngine::Instance().GetDefaultDeviceID();
    }
    Check(b200sv_create((int)deviceID, (int)qBitCount, kPrecision, &sv));
    if (!qubitCount) {
        runningNorm = ZERO_R1; // reference QEngineCPU ctor -> ZeroAmplitudes(), state.cpp:50-54
        return;
    }
    // reference state.cpp:56-63
    const complex ph = (phaseFac == CMPLX_DEFAULT_ARG) ? GetNonunitaryPhase() : phaseFac;
    Check(b200sv_set_permutation(sv, (uint64_t)(bitCapIntOcl)initState, (double)real(ph), (double)imag(ph)));
}

void QEngineCUDA::Copy(QEngineCUDAPtr orig)
{
    QEngine::Copy(std::dynamic_pointer_cast<QEngine>(orig));
    int have = 0;
    Check(b200sv_qubit_count(sv, &have));
    if (have != (int)qubitCount) {
        ResizeZero(qubitCount);
    }
    if (orig->IsZeroAmplitude()) {
        Check(b200sv_zero(sv));
    } else {
        Check(b200sv_copy_state(sv, orig->sv));
    }
}

QEngineCUDA::~QEngineCUDA()
{
    if (sv) {
        b200sv_destroy(sv);
        sv = nullptr;
    }
}

void QEngineCUDA::SetDevice(int64_t dID)
{
    if (dID < 0) {
        dID = (int64_t)CUDAEngine::Instance().GetDefaultDeviceID();
    }
    Check(b200sv_set_device(sv, (int)dID));
    deviceID = dID;
}

bitCapIntOcl QEngineCUDA::GetMaxSize()
{
    return CUDAEngine::Instance().GetDeviceContextPtr(deviceID)->GetMaxAlloc() / sizeof(complex);
}

void QEngineCUDA::ResizeZero(bitLenInt qb)
{
    b200sv_state* n = nullptr;
    Check(b200sv_create((int)deviceID, (int)qb, kPrecision, &n));
    if (sv) {
        b200sv_destroy(sv);
    }
    sv = n;
}

/// QEngine::SetQubitCount is how QPager::MakeEngine (src/qpager.cpp:287-296) and QEngine::Decompose
/// (qengine.hpp:287-293) size an EMPTY engine.  After Compose/Decompose the core already has the new width.
void QEngineCUDA::SetQubitCount(bitLenInt qb)
{
    QEngine::SetQubitCount(qb);
    if (svCountSynced) {
        svCountSynced = false;
        return;
    }
    int have = 0;
    Check(b200sv_qubit_count(sv, &have));
    if (have != (int)qb) {
        ResizeZero(qb);
    }
}

void QEngineCUDA::SyncQubitCount()
{
    int have = 0;
    Check(b200sv_qubit_count(sv, &have));
    svCountSynced = true;
    SetQubitCount((bitLenInt)have);
}

void QEngineCUDA::Finish() { Check(b200sv_finish(sv)); }
bool QEngineCUDA::isFinished()
{
    Check(b200sv_flush(sv));
    return true;
}

// ---- page / buffer ops (reference state.cpp:66-185) -------------------------------------------------------------------

void QEngineCUDA::ZeroAmplitudes()
{
    Check(b200sv_zero(sv));
    runningNorm = ZERO_R1;
}

bool QEngineCUDA::IsZeroAmplitude()
{
    int z = 0;
    Check(b200sv_is_zero(sv, &z));
    return z != 0;
}

void QEngineCUDA::CopyStateVec(QEnginePtr src)
{
    if (qubitCount != src->GetQubitCount()) {
        throw std::invalid_argument("QEngineCUDA::CopyStateVec argument size differs from this!");
    }
    if (src->IsZeroAmplitude()) {
        return ZeroAmplitudes();
    }
    QEngineCUDAPtr c = std::dynamic_pointer_cast<QEngineCUDA>(src);
    if (c) {
        Check(b200sv_copy_state(sv, c->sv));
    } else {
        // e.g. QHybrid switching from QEngineCPU (src/qhybrid.cpp:45-57): stage through the host
        std::unique_ptr<complex[]> tmp(new complex[maxQPowerOcl]);
        src->GetQuantumState(tmp.get());
        Check(b200sv_set_state(sv, tmp.get()));
    }
    runningNorm = (real1)src->GetRunningNorm();
}

void QEngineCUDA::GetAmplitudePage(complex* pagePtr, bitCapIntOcl offset, bitCapIntOcl length)
{
    if (isBadPermRange(offset, length, maxQPowerOcl)) {
        throw std::invalid_argument("QEngineCUDA::GetAmplitudePage range is out-of-bounds!");
    }
    Check(b200sv_get_page(sv, pagePtr, offset, length));
}

void QEngineCUDA::SetAmplitudePage(const complex* pagePtr, bitCapIntOcl offset, bitCapIntOcl length)
{
    if (isBadPermRange(offset, length, maxQPowerOcl)) {
        throw std::invalid_argument("QEngineCUDA::SetAmplitudePage range is out-of-bounds!");
    }
    Check(b200sv_set_page(sv, pagePtr, offset, length));
    if (doNormalize) {
        runningNorm = REAL1_DEFAULT_ARG;
    }
}

void QEngineCUDA::SetAmplitudePage(QEnginePtr pageEnginePtr, bitCapIntOcl srcOffset, bitCapIntOcl dstOffset, bitCapIntOcl length)
{
    if (isBadPermRange(dstOffset, length, maxQPowerOcl)) {
        throw std::invalid_argument("QEngineCUDA::SetAmplitudePage source range is out-of-bounds!");
    }
    QEngineCUDAPtr c = std::dynamic_pointer_cast<QEngineCUDA>(pageEnginePtr);
    if (c) {
        if (isBadPermRange(srcOffset, length, c->maxQPowerOcl)) {
            throw std::invalid_argument("QEngineCUDA::SetAmplitudePage source range is out-of-bounds!");
        }
        Check(b200sv_copy_page(sv, c->sv, srcOffset, dstOffset, length));
    } else {
        std::unique_ptr<complex[]> tmp(new complex[length]);
        pageEnginePtr->GetAmplitudePage(tmp.get(), srcOffset, length);
        Check(b200sv_set_page(sv, tmp.get(), dstOffset, length));
    }
    runningNorm = REAL1_DEFAULT_ARG;
}

void QEngineCUDA::ShuffleBuffers(QEnginePtr engine)
{
    if (qubitCount != engine->GetQubitCount()) {
        throw std::invalid_argument("QEngineCUDA::ShuffleBuffers argument size differs from this!");
    }
    QEngineCUDAPtr c = Cast(engine, "ShuffleBuffers");
    Check(b200sv_shuffle(sv, c->sv));
    runningNorm = REAL1_DEFAULT_ARG;
    c->runningNorm = REAL1_DEFAULT_ARG;
}

QEnginePtr QEngineCUDA::CloneEmpty()
{
    // reference utility.cpp:36-44
    QEngineCUDAPtr c = std::make_shared<QEngineCUDA>(0U, ZERO_BCI, rand_generator, ONE_CMPLX, doNormalize, randGlobalPhase,
        useHostRam, deviceID, !hardware_rand_generator ? false : true, false, (real1_f)amplitudeFloor);
    c->SetQubitCount(qubitCount);
    return c;
}

QInterfacePtr QEngineCUDA::Clone()
{
    // reference utility.cpp:17-34
    QEngineCUDAPtr c = std::dynamic_pointer_cast<QEngineCUDA>(CloneEmpty());
    if (!IsZeroAmplitude()) {
        Check(b200sv_copy_state(c->sv, sv));
    }
    c->runningNorm = runningNorm;
    return c;
}

// ---- state access (reference state.cpp:187-351) -----------------------------------------------------------------------

void QEngineCUDA::SetQuantumState(const complex* inputState)
{
    Check(b200sv_set_state(sv, inputState));
    runningNorm = REAL1_DEFAULT_ARG;
}

void QEngineCUDA::GetQuantumState(complex* outputState)
{
    if (doNormalize) {
        NormalizeState();
    }
    Check(b200sv_get_state(sv, outputState));
}

void QEngineCUDA::GetProbs(real1* outputProbs)
{
    if (doNormalize) {
        NormalizeState();
    }
    Check(b200sv_get_probs(sv, outputProbs));
}

complex QEngineCUDA::GetAmplitude(const bitCapInt& perm)
{
    if (perm >= maxQPower) {
        throw std::invalid_argument("QEngineCUDA::GetAmplitude argument out-of-bounds!");
    }
    double re = 0, im = 0;
    Check(b200sv_get_amplitude(sv, (uint64_t)(bitCapIntOcl)perm, &re, &im));
    return complex((real1)re, (real1)im);
}

void QEngineCUDA::SetAmplitude(const bitCapInt& perm, const complex& amp)
{
    if (perm >= maxQPower) {
        throw std::invalid_argument("QEngineCUDA::SetAmplitude argument out-of-bounds!");
    }
    if (IsZeroAmplitude() && !norm(amp)) {
        return;
    }
    if (runningNorm != REAL1_DEFAULT_ARG) {
        runningNorm += norm(amp) - norm(GetAmplitude(perm));
    }
    Check(b200sv_set_amplitude(sv, (uint64_t)(bitCapIntOcl)perm, (double)real(amp), (double)imag(amp)));
}

void QEngineCUDA::SetPermutation(const bitCapInt& perm, const complex& phaseFac)
{
    // reference state.cpp:228-254
    complex phase;
    if (phaseFac == CMPLX_DEFAULT_ARG) {
        if (randGlobalPhase) {
            const real1_f angle = Rand() * 2 * (real1_f)PI_R1;
            phase = complex((real1)cos(angle), (real1)sin(angle));
        } else {
            phase = ONE_CMPLX;
        }
    } else {
        phase = phaseFac / (real1)abs(phaseFac);
    }
    Check(b200sv_set_permutation(sv, (uint64_t)(bitCapIntOcl)perm, (double)real(phase), (double)imag(phase)));
    runningNorm = ONE_R1;
}

// ---- the gate hot path -----------------------------------------------------------------------------------------------

void QEngineCUDA::Apply2x2(bitCapInt offset1, bitCapInt offset2, const complex* mtrx, bitLenInt bitCount,
    bitCapInt const* qPowersSorted, bool doCalcNorm, real1_f nrm_thresh)
{
    // host part of QEngineCPU::Apply2x2, reference state.cpp:392-431 and :514-531
    if (IsZeroAmplitude()) {
        return;
    }
    if ((offset1 >= maxQPower) || (offset2 >= maxQPower)) {
        throw std::invalid_argument(
            "QEngineCUDA::Apply2x2 offset1 and offset2 parameters must be within allocated qubit bounds!");
    }
    uint64_t pows[64];
    for (bitLenInt i = 0U; i < bitCount; ++i) {
        if (qPowersSorted[i] >= maxQPower) {
            throw std::invalid_argument(
                "QEngineCUDA::Apply2x2 parameter qPowsSorted array values must be within allocated qubit bounds!");
        }
        if (i && (qPowersSorted[i - 1U] == qPowersSorted[i])) {
            throw std::invalid_argument("QEngineCUDA::Apply2x2 parameter qPowSorted array values cannot be "
                                        "duplicated (for control and target qubits)!");
        }
        pows[i] = (uint64_t)(bitCapIntOcl)qPowersSorted[i];
    }
    const bool doApplyNorm = doNormalize && (bitCount == 1U) && (runningNorm > ZERO_R1);
    doCalcNorm &= doApplyNorm || (runningNorm <= ZERO_R1);
    const real1 nrm = doApplyNorm ? ONE_R1 / (real1)sqrt(runningNorm) : ONE_R1;
    if (doCalcNorm) {
        runningNorm = ONE_R1;
    }
    const real1_f thresh = (nrm_thresh < ZERO_R1) ? (real1_f)amplitudeFloor : nrm_thresh;
    double m8[8];
    for (int k = 0; k < 4; ++k) {
        m8[2 * k] = (double)real(mtrx[k]);
        m8[2 * k + 1] = (double)imag(mtrx[k]);
    }
    double normOut = 0;
    Check(b200sv_apply2x2(sv, (uint64_t)(bitCapIntOcl)offset1, (uint64_t)(bitCapIntOcl)offset2, m8, (int)bitCount, pows,
        (double)nrm, doCalcNorm ? (double)thresh : 0.0, doCalcNorm ? &normOut : nullptr));
    if (doApplyNorm) {
        runningNorm = ONE_R1;
    }
    if (doCalcNorm) {
        runningNorm = (real1)normOut;
        if (runningNorm <= FP_NORM_EPSILON) {
            ZeroAmplitudes();
        }
    }
}

void QEngineCUDA::ApplyM(const bitCapInt& regMask, const bitCapInt& result, const complex& nrm)
{
    if (IsZeroAmplitude()) {
        return;
    }
    Check(b200sv_apply_m(sv, (uint64_t)(bitCapIntOcl)regMask, (uint64_t)(bitCapIntOcl)result, (double)real(nrm), (double)imag(nrm)));
    runningNorm = ONE_R1;
}

void QEngineCUDA::XMask(const bitCapInt& mask)
{
    // reference state.cpp:965-1007
    if (mask >= maxQPower) {
        throw std::invalid_argument("QEngineCUDA::XMask mask out-of-bounds!");
    }
    if (IsZeroAmplitude() || (bi_compare_0(mask) == 0)) {
        return;
    }
    if (isPowerOfTwo(mask)) {
        return X(log2(mask));
    }
    Check(b200sv_xmask(sv, (uint64_t)(bitCapIntOcl)mask));
}

void QEngineCUDA::PhaseParity(real1_f radians, const bitCapInt& mask)
{
    // reference state.cpp:1009-1054
    if (mask >= maxQPower) {
        throw std::invalid_argument("QEngineCUDA::PhaseParity mask out-of-bounds!");
    }
    if (IsZeroAmplitude() || (bi_compare_0(mask) == 0)) {
        return;
    }
    if (isPowerOfTwo(mask)) {
        const complex phaseFac = std::polar(ONE_R1, (real1)(radians / 2));
        return Phase(ONE_CMPLX / phaseFac, phaseFac, log2(mask));
    }
    Check(b200sv_phase_parity(sv, (double)radians, (uint64_t)(bitCapIntOcl)mask));
}

void QEngineCUDA::PhaseRootNMask(bitLenInt n, const bitCapInt& mask)
{
    // reference state.cpp:1056-1092
    if (mask >= maxQPower) {
        throw std::invalid_argument("QEngineCUDA::PhaseRootNMask mask out-of-bounds!");
    }
    if (IsZeroAmplitude() || !n || (bi_compare_0(mask) == 0)) {
        return;
    }
    if (n == 1U) {
        return ZMask(mask);
    }
    const real1_f radians = -PI_R1 / pow2Ocl(n - 1U);
    if (isPowerOfTwo(mask)) {
        return Phase(ONE_CMPLX, std::polar(ONE_R1, (real1)radians), log2(mask));
    }
    Check(b200sv_phase_root_n_mask(sv, (int)n, (uint64_t)(bitCapIntOcl)mask));
}

void QEngineCUDA::UniformlyControlledSingleBit(const std::vector<bitLenInt>& controls, bitLenInt qubitIndex, const complex* mtrxs,
    const std::vector<bitCapInt>& mtrxSkipPowers, const bitCapInt& mtrxSkipValueMask)
{
    // reference state.cpp:1094-1198
    if (IsZeroAmplitude()) {
        return;
    }
    if (controls.empty()) {
        return Mtrx(mtrxs + ((bitCapIntOcl)mtrxSkipValueMask * 4U), qubitIndex);
    }
    if (qubitIndex >= qubitCount) {
        throw std::invalid_argument("QEngineCUDA::UniformlyControlledSingleBit qubitIndex is out-of-bounds!");
    }
    ThrowIfQbIdArrayIsBad(controls, qubitCount, "QEngineCUDA::UniformlyControlledSingleBit control is out-of-bounds!");
    std::vector<int> ctrl(controls.begin(), controls.end());
    std::vector<uint64_t> skip(mtrxSkipPowers.size());
    for (size_t i = 0; i < skip.size(); ++i) {
        skip[i] = (uint64_t)(bitCapIntOcl)mtrxSkipPowers[i];
    }
    const size_t nMtrx = (size_t)4U << (controls.size() + mtrxSkipPowers.size());
    std::vector<double> m(2U * nMtrx);
    for (size_t i = 0; i < nMtrx; ++i) {
        m[2 * i] = (double)real(mtrxs[i]);
        m[2 * i + 1] = (double)imag(mtrxs[i]);
    }
    const real1 nrm = (runningNorm > ZERO_R1) ? ONE_R1 / (real1)sqrt(runningNorm) : ONE_R1;
    const bool useNrm = doNormalize && ((ONE_R1 - nrm) > FP_NORM_EPSILON);
    Check(b200sv_uniformly_controlled(sv, (int)ctrl.size(), ctrl.data(), (int)qubitIndex, m.data(), (int)skip.size(), skip.data(),
        (uint64_t)(bitCapIntOcl)mtrxSkipValueMask, useNrm ? (double)nrm : 1.0));
    if (doNormalize) {
        runningNorm = ONE_R1;
    }
}

void QEngineCUDA::UniformParityRZ(const bitCapInt& mask, real1_f angle)
{
    if (mask >= maxQPower) {
        throw std::invalid_argument("QEngineCUDA::UniformParityRZ mask out-of-bounds!");
    }
    if (IsZeroAmplitude()) {
        return;
    }
    Check(b200sv_uniform_parity_rz(sv, 0U, (uint64_t)(bitCapIntOcl)mask, (double)angle));
}

void QEngineCUDA::CUniformParityRZ(const std::vector<bitLenInt>& controls, const bitCapInt& mask, real1_f angle)
{
    if (controls.empty()) {
        return UniformParityRZ(mask, angle);
    }
    if (mask >= maxQPower) {
        throw std::invalid_argument("QEngineCUDA::CUniformParityRZ mask out-of-bounds!");
    }
    ThrowIfQbIdArrayIsBad(controls, qubitCount, "QEngineCUDA::CUniformParityRZ control is out-of-bounds!");
    if (IsZeroAmplitude()) {
        return;
    }
    uint64_t cm = 0;
    for (const bitLenInt& c : controls) {
        cm |= pow2Ocl(c);
    }
    // QEngineCPU's parity runs over an index whose control bits are cleared (state.cpp:1239-1261): a control inside the mask
    // does not count
    Check(b200sv_uniform_parity_rz(sv, cm, (uint64_t)(bitCapIntOcl)mask & ~cm, (double)angle));
}

// ---- probabilities / measurement (reference state.cpp:1751-2107) ---------------------------------------------------

real1_f QEngineCUDA::Prob(bitLenInt qubit)
{
    if (qubit >= qubitCount) {
        throw std::invalid_argument("QEngineCUDA::Prob qubit index parameter must be within allocated qubit bounds!");
    }
    if (doNormalize) {
        NormalizeState();
    }
    if (IsZeroAmplitude()) {
        return ZERO_R1_F;
    }
    double out = 0;
    const uint64_t p = pow2Ocl(qubit);
    Check(b200sv_prob_mask(sv, p, p, &out));
    return clampProb((real1_f)(real1)out);
}

real1_f QEngineCUDA::CtrlOrAntiProb(bool controlState, bitLenInt control, bitLenInt target)
{
    if (IsZeroAmplitude()) {
        return ZERO_R1_F;
    }
    real1_f controlProb = Prob(control);
    if (!controlState) {
        controlProb = ONE_R1 - controlProb;
    }
    if (controlProb <= FP_NORM_EPSILON) {
        return ZERO_R1;
    }
    if ((ONE_R1 - controlProb) <= FP_NORM_EPSILON) {
        return Prob(target);
    }
    if (target >= qubitCount) {
        throw std::invalid_argument(
            "QEngineCUDA::CtrlOrAntiProb target index parameter must be within allocated qubit bounds!");
    }
    double out = 0;
    const uint64_t cp = pow2Ocl(control), tp = pow2Ocl(target);
    Check(b200sv_prob_mask(sv, cp | tp, (controlState ? cp : 0U) | tp, &out));
    return clampProb((real1_f)((real1)out / (real1)controlProb));
}

real1_f QEngineCUDA::ProbReg(bitLenInt start, bitLenInt length, const bitCapInt& permutation)
{
    if (doNormalize) {
        NormalizeState();
    }
    if (IsZeroAmplitude()) {
        return ZERO_R1_F;
    }
    double out = 0;
    Check(b200sv_prob_mask(sv, bitRegMaskOcl(start, length), (uint64_t)(bitCapIntOcl)permutation << start, &out));
    return clampProb((real1_f)(real1)out);
}

real1_f QEngineCUDA::ProbMask(const bitCapInt& mask, const bitCapInt& permutation)
{
    if (mask >= maxQPower) {
        throw std::invalid_argument("QEngineCUDA::ProbMask mask out-of-bounds!");
    }
    if (doNormalize) {
        NormalizeState();
    }
    if (IsZeroAmplitude()) {
        return ZERO_R1_F;
    }
    double out = 0;
    Check(b200sv_prob_mask(sv, (uint64_t)(bitCapIntOcl)mask, (uint64_t)(bitCapIntOcl)permutation, &out));
    return clampProb((real1_f)(real1)out);
}

void QEngineCUDA::ProbMaskAll(const bitCapInt& mask, real1* probsArray)
{
    if (mask >= maxQPower) {
        throw std::invalid_argument("QEngineCUDA::ProbMaskAll mask out-of-bounds!");
    }
    if (doNormalize) {
        NormalizeState();
    }
    Check(b200sv_prob_mask_all(sv, (uint64_t)(bitCapIntOcl)mask, probsArray));
}

void QEngineCUDA::ProbRegAll(bitLenInt start, bitLenInt length, real1* probsArray)
{
    ProbMaskAll(bitCapInt(bitRegMaskOcl(start, length)), probsArray);
}

void QEngineCUDA::ProbBitsAll(const std::vector<bitLenInt>& bits, real1* probsArray)
{
    ThrowIfQbIdArrayIsBad(bits, qubitCount, "QEngineCUDA::ProbBitsAll parameter bits array values must be within allocated qubit bounds!");
    // one device sweep: histogram over the mask in ascending qubit order, then the host permutes its 2^k entries
    bitCapIntOcl mask = 0U;
    for (const bitLenInt& b : bits) {
        mask |= pow2Ocl(b);
    }
    std::vector<bitLenInt> order(bits);
    std::sort(order.begin(), order.end());
    const bitCapIntOcl len = pow2Ocl(bits.size());
    if (order == bits) {
        ProbMaskAll(bitCapInt(mask), probsArray);
        return;
    }
    std::vector<real1> asc((size_t)len);
    ProbMaskAll(bitCapInt(mask), asc.data());
    std::vector<bitLenInt> pos(bits.size());
    for (size_t p = 0U; p < bits.size(); ++p) {
        pos[p] = (bitLenInt)(std::find(order.begin(), order.end(), bits[p]) - order.begin());
    }
    for (bitCapIntOcl i = 0U; i < len; ++i) {
        bitCapIntOcl src = 0U;
        for (size_t p = 0U; p < bits.size(); ++p) {
            if ((i >> p) & 1U) {
                src |= pow2Ocl(pos[p]);
            }
        }
        probsArray[i] = asc[(size_t)src];
    }
}

static void SampleShots(QEngineCUDA* eng, b200sv_t sv, const std::vector<bitCapInt>& qPowers, unsigned shots, bitLenInt qubitCount,
    std::vector<bitCapIntOcl>& keys)
{
    std::vector<bitLenInt> bitMap(qPowers.size());
    std::transform(qPowers.begin(), qPowers.end(), bitMap.begin(), log2);
    ThrowIfQbIdArrayIsBad(bitMap, qubitCount,
        "QInterface::MultiShotMeasureMask parameter qPowers array values must be within allocated qubit bounds!");
    keys.assign(shots, 0U);
    std::vector<double> rnds(shots);
    for (unsigned i = 0U; i < shots; ++i) {
        rnds[i] = (double)eng->Rand();
    }
    if (bitMap.size() <= 16U) {
        // few measured qubits: the 2^k histogram in one sweep, host draws (what QEngine::MultiShotMeasureMask does)
        const bitCapIntOcl len = pow2Ocl(bitMap.size());
        std::vector<real1> probs((size_t)len);
        eng->ProbBitsAll(bitMap, probs.data());
        std::vector<double> cum((size_t)len);
        double tot = 0;
        for (bitCapIntOcl i = 0U; i < len; ++i) {
            tot += (double)probs[(size_t)i];
            cum[(size_t)i] = tot;
        }
        for (unsigned i = 0U; i < shots; ++i) {
            const double r = rnds[i] * tot;
            bitCapIntOcl k = (bitCapIntOcl)(std::upper_bound(cum.begin(), cum.end(), r) - cum.begin());
            keys[i] = (k < len) ? k : (len - 1U);
        }
        return;
    }
    std::vector<uint64_t> perms(shots);
    if (b200sv_sample_many(sv, (int)shots, rnds.data(), perms.data()) != B200SV_OK) {
        throw std::runtime_error(std::string("QEngineCUDA::MultiShotMeasureMask: ") + b200sv_last_error());
    }
    for (unsigned i = 0U; i < shots; ++i) {
        bitCapIntOcl key = 0U;
        for (size_t p = 0U; p < bitMap.size(); ++p) {
            if ((perms[i] >> bitMap[p]) & 1U) {
                key |= pow2Ocl(p);
            }
        }
        keys[i] = key;
    }
}

std::map<bitCapInt, int> QEngineCUDA::MultiShotMeasureMask(const std::vector<bitCapInt>& qPowers, unsigned shots)
{
    std::map<bitCapInt, int> results;
    if (!shots) {
        return results;
    }
    if (doNormalize) {
        NormalizeState();
    }
    std::vector<bitCapIntOcl> keys;
    SampleShots(this, sv, qPowers, shots, qubitCount, keys);
    for (const bitCapIntOcl& k : keys) {
        ++results[bitCapInt(k)];
    }
    return results;
}

void QEngineCUDA::MultiShotMeasureMask(const std::vector<bitCapInt>& qPowers, unsigned shots, unsigned long long* shotsArray)
{
    if (!shots) {
        return;
    }
    if (doNormalize) {
        NormalizeState();
    }
    std::vector<bitCapIntOcl> keys;
    SampleShots(this, sv, qPowers, shots, qubitCount, keys);
    for (unsigned i = 0U; i < shots; ++i) {
        shotsArray[i] = (unsigned long long)keys[i];
    }
}

real1_f QEngineCUDA::ProbParity(const bitCapInt& mask)
{
    if (mask >= maxQPower) {
        throw std::invalid_argument("QEngineCUDA::ProbParity mask out-of-bounds!");
    }
    if (doNormalize) {
        NormalizeState();
    }
    if (IsZeroAmplitude() || (bi_compare_0(mask) == 0)) {
        return ZERO_R1_F;
    }
    double out = 0;
    Check(b200sv_prob_parity(sv, (uint64_t)(bitCapIntOcl)mask, &out));
    return clampProb((real1_f)(real1)out);
}

bool QEngineCUDA::ForceMParity(const bitCapInt& mask, bool result, bool doForce)
{
    if (mask >= maxQPower) {
        throw std::invalid_argument("QEngineCUDA::ForceMParity mask out-of-bounds!");
    }
    if (IsZeroAmplitude() || (bi_compare_0(mask) == 0)) {
        return false;
    }
    if (!doForce) {
        result = (Rand() <= ProbParity(mask));
    }
    double kept = 0;
    Check(b200sv_collapse_parity(sv, (uint64_t)(bitCapIntOcl)mask, result ? 1 : 0, &kept));
    runningNorm = (real1)kept;
    if (!doNormalize) {
        NormalizeState();
    }
    return result;
}

bitCapInt QEngineCUDA::HighestProbAll()
{
    if (IsZeroAmplitude()) {
        return ZERO_BCI; // reference src/qengine/cuda.cu:2906-2912
    }
    uint64_t perm = 0U;
    Check(b200sv_highest_prob(sv, &perm));
    return bitCapInt((bitCapIntOcl)perm);
}

std::vector<bitCapInt> QEngineCUDA::HighestProbAll(size_t n)
{
    // the reference's edge rules (qinterface.cpp:962-973); the selection itself is exact, without the early exit on the
    // running sum (INTEGRATION.md)
    if (!n) {
        return std::vector<bitCapInt>();
    }
    if (n == 1U) {
        return std::vector<bitCapInt>{ HighestProbAll() };
    }
    if (bitCapInt((bitCapIntOcl)n) > maxQPower) {
        throw std::invalid_argument("QInterface::HighestProbAll(n) requested more !");
    }
    if (doNormalize) {
        NormalizeState();
    }
    std::vector<uint64_t> perms(n);
    Check(b200sv_highest_probs(sv, (uint64_t)n, perms.data()));
    std::vector<bitCapInt> out(n);
    for (size_t t = 0U; t < n; ++t) {
        out[t] = bitCapInt((bitCapIntOcl)perms[t]);
    }
    return out;
}

static bool LossyOnDevice(int p, int b) { return (p >= 1) && (p <= 6) && (b >= 1) && (b <= 16); }

void QEngineCUDA::LossySaveStateVector(std::string f, int p, int b)
{
    // QEngineCUDA (cuda.cu:3017-3035) / QEngineCPU (state.cpp:256-272): normalise first, p = 0 means p = qubitCount
    if (!p) {
        p = (int)qubitCount;
    }
    if (!LossyOnDevice(p, b)) {
        return QInterface::LossySaveStateVector(f, p, b);
    }
    if (doNormalize) {
        NormalizeState();
    }
    std::random_device rd;
    const uint64_t seed = ((uint64_t)rd() << 32U) | (uint64_t)rd();
    Check(b200sv_lossy_save(sv, f.c_str(), p, b, seed));
}

void QEngineCUDA::LossyLoadStateVector(std::string f)
{
    if (doNormalize) {
        NormalizeState();
    }
    if (!std::ifstream(f).good()) {
        // QEngineCPU (state.cpp:284-289) drops its state; the reference's CUDA engine would read garbage
        return ZeroAmplitudes();
    }
    int nq = 0, p = 0, b = 0;
    Check(b200sv_lossy_probe(f.c_str(), (int)(8U * sizeof(real1)), &nq, &p, &b));
    if (!LossyOnDevice(p, b)) {
        return QInterface::LossyLoadStateVector(f);
    }
    if ((bitLenInt)nq > qubitCount) {
        Allocate(qubitCount, (bitLenInt)nq - qubitCount);
    } else if ((bitLenInt)nq < qubitCount) {
        Dispose(0U, qubitCount - (bitLenInt)nq);
    }
    Check(b200sv_lossy_load(sv, f.c_str()));
    runningNorm = REAL1_DEFAULT_ARG;
}

bitCapInt QEngineCUDA::MAll()
{
    // QEngineCPU::MAll (state.cpp:2026-2050) with the cumulative search done on the device
    const real1_f rnd = Rand();
    if (doNormalize) {
        NormalizeState();
    }
    uint64_t perm = 0;
    Check(b200sv_sample(sv, (double)rnd, &perm));
    SetPermutation(bitCapInt(perm));
    return bitCapInt(perm);
}

real1_f QEngineCUDA::GetExpectation(bitLenInt valueStart, bitLenInt valueLength)
{
    double avg = 0, tot = 0;
    Check(b200sv_expectation(sv, (int)valueStart, (int)valueLength, &avg));
    Check(b200sv_norm(sv, 0.0, &tot));
    return (tot > 0) ? (real1_f)(avg / tot) : (real1_f)avg;
}

// ---- observables (reference src/qinterface/qinterface.cpp:542-806): same checks and messages, same k = 0 / k = 1 branches
// (the base class's, over Prob), and one read-only sweep for k >= 2 --------------------------------------------------------

bool QEngineCUDA::BitsWeights(const std::vector<bitLenInt>& bits, const std::vector<bitCapInt>& perms, const bitCapInt& offset,
    std::vector<int>& b, std::vector<uint64_t>& p, uint64_t& off) const
{
    const bitCapInt max64 = bitCapInt(~(uint64_t)0U);
    if (bi_compare(offset, max64) > 0) {
        return false;
    }
    off = (uint64_t)offset;
    uint64_t top = off;
    b.resize(bits.size());
    p.resize(bits.size() << 1U);
    for (size_t i = 0U; i < bits.size(); ++i) {
        b[i] = (int)bits[i];
        for (size_t e = 0U; e < 2U; ++e) {
            const bitCapInt& v = perms[(i << 1U) | e];
            if (bi_compare(v, max64) > 0) {
                return false;
            }
            p[(i << 1U) | e] = (uint64_t)v;
        }
        const uint64_t m = std::max(p[i << 1U], p[(i << 1U) | 1U]);
        if (m > ~top) {
            return false;
        }
        top += m;
    }
    return true;
}

void QEngineCUDA::Moments(const std::vector<int>& b, const std::vector<uint64_t>& p, uint64_t off, double center, double* out)
{
    if (doNormalize) {
        NormalizeState();
    }
    Check(b200sv_moments_bits(sv, (int)b.size(), b.data(), p.data(), off, center, out));
}

void QEngineCUDA::MomentsFloats(const std::vector<bitLenInt>& bits, const std::vector<real1_f>& weights, double* out)
{
    if (doNormalize) {
        NormalizeState();
    }
    std::vector<int> b(bits.begin(), bits.end());
    std::vector<double> w(weights.begin(), weights.begin() + (bits.size() << 1U));
    Check(b200sv_moments_floats(sv, (int)b.size(), b.data(), w.data(), 0.0, out));
}

real1_f QEngineCUDA::ExpectationBitsFactorized(
    const std::vector<bitLenInt>& bits, const std::vector<bitCapInt>& perms, const bitCapInt& offset)
{
    if (perms.size() < (bits.size() << 1U)) {
        throw std::invalid_argument(
            "QInterface::ExpectationBitsFactorized() must supply at least twice as many 'perms' as bits!");
    }
    ThrowIfQbIdArrayIsBad(bits, qubitCount,
        "QInterface::ExpectationBitsFactorized() parameter qubits vector values must be within allocated qubit "
        "bounds!");
    std::vector<int> b;
    std::vector<uint64_t> p;
    uint64_t off = 0U;
    if ((bits.size() < 2U) || !BitsWeights(bits, perms, offset, b, p, off)) {
        return QEngine::ExpectationBitsFactorized(bits, perms, offset);
    }
    double m[3];
    Moments(b, p, off, 0.0, m);
    return (real1_f)m[1];
}

real1_f QEngineCUDA::VarianceBitsFactorized(
    const std::vector<bitLenInt>& bits, const std::vector<bitCapInt>& perms, const bitCapInt& offset)
{
    if (perms.size() < (bits.size() << 1U)) {
        throw std::invalid_argument(
            "QInterface::VarianceBitsFactorized() must supply at least twice as many 'perms' as bits!");
    }
    ThrowIfQbIdArrayIsBad(bits, qubitCount,
        "QInterface::VarianceBitsFactorized() parameter qubits vector values must be within allocated qubit "
        "bounds!");
    std::vector<int> b;
    std::vector<uint64_t> p;
    uint64_t off = 0U;
    if ((bits.size() < 2U) || !BitsWeights(bits, perms, offset, b, p, off)) {
        return QEngine::VarianceBitsFactorized(bits, perms, offset);
    }
    const real1_f mean = ExpectationBitsFactorized(bits, perms, offset);
    // a second sweep centred on the mean: sum p (w - mean)^2 without the cancellation of E[w^2] - E[w]^2
    double m[3];
    Moments(b, p, off, (double)mean, m);
    return (real1_f)m[2];
}

real1_f QEngineCUDA::ExpectationFloatsFactorized(const std::vector<bitLenInt>& bits, const std::vector<real1_f>& weights)
{
    if (weights.size() < (bits.size() << 1U)) {
        throw std::invalid_argument(
            "QInterface::ExpectationFloatsFactorized() must supply at least twice as many weights as bits!");
    }
    ThrowIfQbIdArrayIsBad(bits, qubitCount,
        "QInterface::ExpectationFloatsFactorized() parameter qubits vector values must be within allocated qubit "
        "bounds!");
    if (bits.size() < 2U) {
        return QEngine::ExpectationFloatsFactorized(bits, weights);
    }
    double m[3];
    MomentsFloats(bits, weights, m);
    return (real1_f)m[1];
}

real1_f QEngineCUDA::VarianceFloatsFactorized(const std::vector<bitLenInt>& bits, const std::vector<real1_f>& weights)
{
    if (weights.size() < (bits.size() << 1U)) {
        throw std::invalid_argument(
            "QInterface::VarianceFloatsFactorized() must supply at least twice as many weights as bits!");
    }
    ThrowIfQbIdArrayIsBad(bits, qubitCount,
        "QInterface::VarianceFloatsFactorized() parameter qubits vector values must be within allocated qubit "
        "bounds!");
    if (bits.size() < 2U) {
        return QEngine::VarianceFloatsFactorized(bits, weights);
    }
    double m[3];
    MomentsFloats(bits, weights, m);
    // the reference sums p (w - mean) UNSQUARED for k >= 2 (qinterface.cpp:653) = mean (1 - S0); kept for parity with
    // QEngineCPU (its 1-bit branch squares; the true variance is S2 centred on the mean)
    const real1_f mean = (real1_f)m[1];
    return (real1_f)(m[1] - (double)mean * m[0]);
}

bool QEngineCUDA::PauliMasks(std::vector<bitLenInt>& bits, const std::vector<Pauli>& paulis, uint64_t& x, uint64_t& z) const
{
    if (paulis.size() < bits.size()) {
        return false;
    }
    // the PauliI-dropping loop of qinterface.cpp:719-726 as written: it re-reads bits.size() after each erase, so some PauliI
    // entries survive it, and those then get the weights (1, -1) without a basis gate — they count as PauliZ
    std::vector<Pauli> ps(paulis.begin(), paulis.begin() + bits.size());
    for (size_t i = 0U; i < bits.size(); ++i) {
        const size_t j = bits.size() - (i + 1U);
        if (ps[j] == PauliI) {
            bits.erase(bits.begin() + j);
            ps.erase(ps.begin() + j);
        }
    }
    x = z = 0U;
    for (size_t i = 0U; i < bits.size(); ++i) {
        if (bits[i] >= qubitCount) {
            return false;
        }
        const uint64_t pw = pow2Ocl(bits[i]);
        if ((x | z) & pw) {
            return false;
        }
        // include/pauli.hpp: X = 1, Z = 2, Y = 3
        if (ps[i] == PauliX || ps[i] == PauliY) {
            x |= pw;
        }
        if (ps[i] != PauliX) {
            z |= pw;
        }
    }
    return true;
}

// ExpectationPauliAll / VariancePauliAll (qinterface.cpp:659-769) rotate each X / Y qubit into the Z basis, run the Floats query
// with weights (1, -1) and rotate back.  b200sv_expectation_pauli returns S0 = sum |psi|^2 and E = <psi|P|psi> without
// touching the state; in the rotated basis Prob(bits[0]) of the 1-bit branch is (S0 - E) / 2 and the k >= 2 sum is E.
real1_f QEngineCUDA::ExpectationPauliAll(std::vector<bitLenInt> bits, std::vector<Pauli> paulis)
{
    std::vector<bitLenInt> kept = bits;
    uint64_t x = 0U, z = 0U;
    if (!PauliMasks(kept, paulis, x, z)) {
        return QEngine::ExpectationPauliAll(bits, paulis);
    }
    if (kept.empty()) {
        return ONE_R1_F;
    }
    if (doNormalize) {
        NormalizeState();
    }
    double o[2];
    Check(b200sv_expectation_pauli(sv, x, z, o));
    if (kept.size() == 1U) {
        const real1_f prob = clampProb((real1_f)((o[0] - o[1]) / 2));
        return (ONE_R1_F - prob) - prob;
    }
    return (real1_f)o[1];
}

real1_f QEngineCUDA::VariancePauliAll(std::vector<bitLenInt> bits, std::vector<Pauli> paulis)
{
    std::vector<bitLenInt> kept = bits;
    uint64_t x = 0U, z = 0U;
    if (!PauliMasks(kept, paulis, x, z)) {
        return QEngine::VariancePauliAll(bits, paulis);
    }
    if (kept.empty()) {
        return ONE_R1_F;
    }
    if (doNormalize) {
        NormalizeState();
    }
    double o[2];
    Check(b200sv_expectation_pauli(sv, x, z, o));
    if (kept.size() == 1U) {
        const real1_f prob = clampProb((real1_f)((o[0] - o[1]) / 2));
        const real1_f mean = (ONE_R1_F - prob) - prob;
        const real1_f var0 = ONE_R1_F - mean;
        const real1_f var1 = -ONE_R1_F - mean;
        return var0 * var0 * (ONE_R1_F - prob) + var1 * var1 * prob;
    }
    // VarianceFloatsFactorized's unsquared k >= 2 sum with weights (1, -1): E - E S0
    const real1_f mean = (real1_f)o[1];
    return (real1_f)(o[1] - (double)mean * o[0]);
}

// the matrix QInterface::U builds (rotational.cpp:18-26), rounded as it rounds
static void UMatrix(real1_f theta, real1_f phi, real1_f lambda, complex* m)
{
    const real1 cos0 = (real1)cos(theta / 2);
    const real1 sin0 = (real1)sin(theta / 2);
    m[0U] = complex(cos0, ZERO_R1);
    m[1U] = sin0 * complex((real1)(-cos(lambda)), (real1)(-sin(lambda)));
    m[2U] = sin0 * complex((real1)cos(phi), (real1)sin(phi));
    m[3U] = cos0 * complex((real1)cos(phi + lambda), (real1)sin(phi + lambda));
}

real1_f QEngineCUDA::BasisMoments(
    bool isExp, const std::vector<bitLenInt>& bits, const complex* mats, std::vector<real1_f> eigenVals)
{
    const size_t k = bits.size();
    if (eigenVals.empty()) {
        for (size_t i = 0U; i < k; ++i) {
            eigenVals.push_back(ONE_R1_F);
            eigenVals.push_back(-ONE_R1_F);
        }
    }
    // the checks of the Floats query the reference runs (qinterface.cpp:620-630, 771-780)
    const std::string what = isExp ? "ExpectationFloatsFactorized" : "VarianceFloatsFactorized";
    if (eigenVals.size() < (k << 1U)) {
        throw std::invalid_argument("QInterface::" + what + "() must supply at least twice as many weights as bits!");
    }
    ThrowIfQbIdArrayIsBad(
        bits, qubitCount, "QInterface::" + what + "() parameter qubits vector values must be within allocated qubit bounds!");
    if (doNormalize) {
        NormalizeState();
    }
    std::vector<int> b(bits.begin(), bits.end());
    std::vector<double> m(k << 3U);
    for (size_t i = 0U; i < (k << 2U); ++i) {
        m[i << 1U] = (double)real(mats[i]);
        m[(i << 1U) | 1U] = (double)imag(mats[i]);
    }
    double o[3];
    if (k == 1U) {
        // the Floats query's 1-bit branch on Prob(bits[0]) of the rotated state: a sweep with weights (0, 1)
        const double w01[2]{ 0.0, 1.0 };
        Check(b200sv_moments_basis(sv, 1, b.data(), m.data(), w01, 0.0, o));
        const real1_f prob = clampProb((real1_f)o[1]);
        const real1_f mean = eigenVals[0U] * (ONE_R1_F - prob) + eigenVals[1U] * prob;
        if (isExp) {
            return mean;
        }
        const real1_f var0 = eigenVals[0U] - mean;
        const real1_f var1 = eigenVals[1U] - mean;
        return var0 * var0 * (ONE_R1_F - prob) + var1 * var1 * prob;
    }
    std::vector<double> w(eigenVals.begin(), eigenVals.begin() + (k << 1U));
    Check(b200sv_moments_basis(sv, (int)k, b.data(), m.data(), w.data(), 0.0, o));
    const real1_f mean = (real1_f)o[1];
    // the reference's k >= 2 variance is the unsquared sum p (w - mean) (qinterface.cpp:653)
    return isExp ? mean : (real1_f)(o[1] - (double)mean * o[0]);
}

real1_f QEngineCUDA::ExpVarUnitaryAll(bool isExp, const std::vector<bitLenInt>& bits,
    const std::vector<std::shared_ptr<complex>>& basisOps, std::vector<real1_f> eigenVals)
{
    if (bits.size() > B200SV_BASIS_MAX_QUBITS) {
        return QEngine::ExpVarUnitaryAll(isExp, bits, basisOps, eigenVals);
    }
    if (bits.empty()) {
        return ONE_R1_F;
    }
    std::vector<complex> mats(bits.size() << 2U);
    for (size_t i = 0U; i < bits.size(); ++i) {
        inv2x2(basisOps[i].get(), mats.data() + (i << 2U));
    }
    return BasisMoments(isExp, bits, mats.data(), eigenVals);
}

real1_f QEngineCUDA::ExpVarUnitaryAll(
    bool isExp, const std::vector<bitLenInt>& bits, const std::vector<real1_f>& basisOps, std::vector<real1_f> eigenVals)
{
    if (bits.size() > B200SV_BASIS_MAX_QUBITS) {
        return QEngine::ExpVarUnitaryAll(isExp, bits, basisOps, eigenVals);
    }
    if (bits.empty()) {
        return ONE_R1_F;
    }
    std::vector<complex> mats(bits.size() << 2U);
    for (size_t i = 0U; i < bits.size(); ++i) {
        const size_t i3 = 3U * i;
        UMatrix(-basisOps[i3], -basisOps[i3 + 1U], -basisOps[i3 + 2U], mats.data() + (i << 2U));
    }
    const real1_f toRet = BasisMoments(isExp, bits, mats.data(), eigenVals);
    for (size_t i = 0U; i < bits.size(); ++i) {
        const size_t i3 = 3U * i;
        complex undo[4U], net[4U];
        UMatrix(basisOps[i3], basisOps[i3 + 1U], basisOps[i3 + 2U], undo);
        mul2x2(undo, mats.data() + (i << 2U), net);
        Mtrx(net, bits[i]);
    }
    return toRet;
}

void QEngineCUDA::GetReducedDensityMatrix(const std::vector<bitLenInt>& qubits, complex* outputState)
{
    std::vector<bool> seen(qubitCount, false);
    for (const bitLenInt q : qubits) {
        if (q >= qubitCount) {
            throw std::invalid_argument("QEngineCUDA::GetReducedDensityMatrix qubit index out of bounds!");
        }
        if (seen[q]) {
            throw std::invalid_argument("QEngineCUDA::GetReducedDensityMatrix repeated qubit index!");
        }
        seen[q] = true;
    }
    if (qubits.size() > B200SV_RDM_MAX_QUBITS) {
        QInterface::GetReducedDensityMatrix(qubits, outputState);
        return;
    }
    // like the base class (GetAmplitude, state.cpp:193) this does not normalise
    const size_t dim = (size_t)1U << qubits.size();
    std::vector<int> q(qubits.begin(), qubits.end());
    std::vector<double> rho(2U * dim * dim);
    Check(b200sv_reduced_density_matrix(sv, (int)q.size(), q.data(), rho.data()));
    for (size_t i = 0U; i < dim * dim; ++i) {
        outputState[i] = complex((real1)rho[2U * i], (real1)rho[2U * i + 1U]);
    }
}

// ---- structure (reference state.cpp:1271-1748, utility.cpp:54-68) --------------------------------------------------

bitLenInt QEngineCUDA::Compose(QEngineCUDAPtr toCopy) { return Compose(toCopy, qubitCount); }

bitLenInt QEngineCUDA::Compose(QEngineCUDAPtr toCopy, bitLenInt start)
{
    if (start > qubitCount) {
        throw std::invalid_argument("QEngineCUDA::Compose start index is out-of-bounds!");
    }
    if (!toCopy->qubitCount) {
        return start;
    }
    if (!qubitCount) {
        // reference state.cpp:1286-1297
        ResizeZero(toCopy->qubitCount);
        QEngine::SetQubitCount(toCopy->qubitCount);
        if (!toCopy->IsZeroAmplitude()) {
            Check(b200sv_copy_state(sv, toCopy->sv));
        }
        runningNorm = toCopy->runningNorm;
        return 0U;
    }
    if (doNormalize) {
        NormalizeState();
    }
    if (toCopy->doNormalize) {
        toCopy->NormalizeState();
    }
    Check(b200sv_compose(sv, toCopy->sv, (int)start));
    SyncQubitCount();
    if (IsZeroAmplitude()) {
        runningNorm = ZERO_R1;
    }
    return start;
}

void QEngineCUDA::Decompose(bitLenInt start, QInterfacePtr destination)
{
    QEngineCUDAPtr dest = Cast(destination, "Decompose");
    const bitLenInt length = dest->GetQubitCount();
    if (isBadBitRange(start, length, qubitCount)) {
        throw std::invalid_argument("QEngineCUDA::DecomposeDispose range is out-of-bounds!");
    }
    if (!length) {
        return;
    }
    if (doNormalize) {
        NormalizeState();
    }
    Check(b200sv_decompose(sv, (int)start, (int)length, dest->sv));
    SyncQubitCount();
    dest->runningNorm = dest->IsZeroAmplitude() ? ZERO_R1 : ONE_R1;
}

void QEngineCUDA::Dispose(bitLenInt start, bitLenInt length)
{
    if (isBadBitRange(start, length, qubitCount)) {
        throw std::invalid_argument("QEngineCUDA::DecomposeDispose range is out-of-bounds!");
    }
    if (!length) {
        return;
    }
    if (doNormalize) {
        NormalizeState();
    }
    Check(b200sv_decompose(sv, (int)start, (int)length, nullptr));
    SyncQubitCount();
}

void QEngineCUDA::Dispose(bitLenInt start, bitLenInt length, const bitCapInt& disposedPerm)
{
    if (isBadBitRange(start, length, qubitCount)) {
        throw std::invalid_argument("QEngineCUDA::Dispose range is out-of-bounds!");
    }
    if (!length) {
        return;
    }
    if (doNormalize) {
        NormalizeState();
    }
    Check(b200sv_dispose_perm(sv, (int)start, (int)length, (uint64_t)(bitCapIntOcl)disposedPerm));
    SyncQubitCount();
}

bitLenInt QEngineCUDA::Allocate(bitLenInt start, bitLenInt length)
{
    if (start > qubitCount) {
        throw std::invalid_argument("QEngineCUDA::Allocate argument is out-of-bounds!");
    }
    if (!length) {
        return start;
    }
    QEngineCUDAPtr nQubits = std::make_shared<QEngineCUDA>(length, ZERO_BCI, rand_generator, ONE_CMPLX, doNormalize,
        randGlobalPhase, useHostRam, deviceID, !hardware_rand_generator ? false : true, false, (real1_f)amplitudeFloor);
    return Compose(nQubits, start);
}

// ---- norm (reference state.cpp:2109-2268) ------------------------------------------------------------------------------

real1_f QEngineCUDA::SumSqrDiff(QInterfacePtr toCompare)
{
    if (!toCompare) {
        return ONE_R1_F;
    }
    if (this == toCompare.get()) {
        return ZERO_R1_F;
    }
    if (qubitCount != toCompare->GetQubitCount()) {
        return ONE_R1_F;
    }
    QEngineCUDAPtr o = Cast(toCompare, "SumSqrDiff");
    if (doNormalize) {
        NormalizeState();
    }
    if (o->doNormalize) {
        o->NormalizeState();
    }
    if (IsZeroAmplitude() && o->IsZeroAmplitude()) {
        return ZERO_R1_F;
    }
    if (IsZeroAmplitude()) {
        o->UpdateRunningNorm();
        return (real1_f)o->runningNorm;
    }
    if (o->IsZeroAmplitude()) {
        UpdateRunningNorm();
        return (real1_f)runningNorm;
    }
    double re = 0, im = 0;
    Check(b200sv_inner(sv, o->sv, &re, &im));
    return ONE_R1_F - clampProb((real1_f)norm(complex((real1)re, (real1)im)));
}

void QEngineCUDA::NormalizeState(real1_f nrm_f, real1_f norm_thresh_f, real1_f phaseArg)
{
    if (IsZeroAmplitude()) {
        return;
    }
    if ((runningNorm == REAL1_DEFAULT_ARG) && (nrm_f == REAL1_DEFAULT_ARG)) {
        UpdateRunningNorm();
    }
    real1 nrm = (real1)nrm_f;
    real1 norm_thresh = (real1)norm_thresh_f;
    if (nrm < ZERO_R1) {
        nrm = runningNorm;
    }
    if (nrm <= FP_NORM_EPSILON) {
        return ZeroAmplitudes();
    }
    if ((abs(ONE_R1 - nrm) <= FP_NORM_EPSILON) && ((phaseArg * phaseArg) <= FP_NORM_EPSILON)) {
        return;
    }
    if (norm_thresh < ZERO_R1) {
        norm_thresh = amplitudeFloor;
    }
    Check(b200sv_normalize(sv, (double)nrm, (double)norm_thresh, (double)phaseArg));
    runningNorm = ONE_R1;
}

void QEngineCUDA::UpdateRunningNorm(real1_f norm_thresh)
{
    if (IsZeroAmplitude()) {
        runningNorm = ZERO_R1;
        return;
    }
    if (norm_thresh < ZERO_R1) {
        norm_thresh = (real1_f)amplitudeFloor;
    }
    double out = 0;
    Check(b200sv_norm(sv, (double)norm_thresh, &out));
    runningNorm = (real1)out;
    if (runningNorm <= FP_NORM_EPSILON) {
        ZeroAmplitudes();
    }
}

// ---- QAlu / ROL: each member is ONE out-of-place basis-map sweep on the device (include/b200sv.h "QAlu family").
// What stays here is what the reference's QEngineCPU does above its loops (src/qengine/arithmetic.cpp): argument
// checks that throw std::invalid_argument, the trivial-argument shortcuts, and the SetReg / M / X pre-steps.

uint64_t QEngineCUDA::CtrlMask(const std::vector<bitLenInt>& controls, const char* what) const
{
    uint64_t m = 0U;
    for (const bitLenInt c : controls) {
        if (c >= qubitCount) {
            throw std::invalid_argument(std::string("QEngineCUDA::") + what + " control is out-of-bounds!");
        }
        m |= pow2Ocl(c);
    }
    return m;
}

void QEngineCUDA::ROL(bitLenInt shift, bitLenInt start, bitLenInt length)
{
    Check(b200sv_rol(sv, (int)shift, (int)start, (int)length));
}

void QEngineCUDA::ROR(bitLenInt shift, bitLenInt start, bitLenInt length)
{
    if (!length) {
        return;
    }
    shift %= length;
    if (shift) {
        ROL(length - shift, start, length);
    }
}

#if ENABLE_ALU
#define U64(x) ((uint64_t)(bitCapIntOcl)(x))
void QEngineCUDA::INC(const bitCapInt& toAdd, bitLenInt start, bitLenInt length)
{
    Check(b200sv_inc(sv, U64(toAdd), (int)start, (int)length, 0U));
}
void QEngineCUDA::CINC(const bitCapInt& toAdd, bitLenInt start, bitLenInt length, const std::vector<bitLenInt>& controls)
{
    Check(b200sv_inc(sv, U64(toAdd), (int)start, (int)length, CtrlMask(controls, "CINC")));
}
void QEngineCUDA::INCDECC(const bitCapInt& toMod, bitLenInt start, bitLenInt length, bitLenInt carryIndex)
{
    Check(b200sv_incdecc(sv, U64(toMod), (int)start, (int)length, (int)carryIndex));
}
void QEngineCUDA::INCS(const bitCapInt& toAdd, bitLenInt start, bitLenInt length, bitLenInt overflowIndex)
{
    Check(b200sv_incs(sv, U64(toAdd), (int)start, (int)length, (int)overflowIndex));
}
void QEngineCUDA::INCDECSC(const bitCapInt& toMod, bitLenInt start, bitLenInt length, bitLenInt carryIndex)
{
    Check(b200sv_incdecsc(sv, U64(toMod), (int)start, (int)length, -1, (int)carryIndex));
}
void QEngineCUDA::INCDECSC(const bitCapInt& toMod, bitLenInt start, bitLenInt length, bitLenInt overflowIndex, bitLenInt carryIndex)
{
    Check(b200sv_incdecsc(sv, U64(toMod), (int)start, (int)length, (int)overflowIndex, (int)carryIndex));
}
void QEngineCUDA::PhaseFlipIfLess(const bitCapInt& greaterPerm, bitLenInt start, bitLenInt length)
{
    Check(b200sv_phase_flip_if_less(sv, U64(greaterPerm), (int)start, (int)length, -1));
}
void QEngineCUDA::CPhaseFlipIfLess(const bitCapInt& greaterPerm, bitLenInt start, bitLenInt length, bitLenInt flagIndex)
{
    Check(b200sv_phase_flip_if_less(sv, U64(greaterPerm), (int)start, (int)length, (int)flagIndex));
}

// MUL / DIV and controlled forms: arithmetic.cpp:458-485, 553-593
void QEngineCUDA::MUL(const bitCapInt& toMul, bitLenInt start, bitLenInt carryStart, bitLenInt length)
{
    SetReg(carryStart, length, ZERO_BCI);
    if (bi_compare_0(toMul) == 0) {
        return SetReg(start, length, ZERO_BCI);
    }
    if (bi_compare_1(toMul) == 0) {
        return;
    }
    Check(b200sv_muldiv(sv, 0, U64(toMul), (int)start, (int)carryStart, (int)length, 0U));
}
void QEngineCUDA::DIV(const bitCapInt& toDiv, bitLenInt start, bitLenInt carryStart, bitLenInt length)
{
    if (bi_compare_0(toDiv) == 0) {
        throw std::runtime_error("DIV by zero");
    }
    if (bi_compare_1(toDiv) == 0) {
        return;
    }
    Check(b200sv_muldiv(sv, 1, U64(toDiv), (int)start, (int)carryStart, (int)length, 0U));
}
void QEngineCUDA::CMUL(const bitCapInt& toMul, bitLenInt start, bitLenInt carryStart, bitLenInt length,
    const std::vector<bitLenInt>& controls)
{
    if (controls.empty()) {
        return MUL(toMul, start, carryStart, length);
    }
    SetReg(carryStart, length, ZERO_BCI);
    if (bi_compare_0(toMul) == 0) {
        return SetReg(start, length, ZERO_BCI);
    }
    if (bi_compare_1(toMul) == 0) {
        return;
    }
    Check(b200sv_muldiv(sv, 0, U64(toMul), (int)start, (int)carryStart, (int)length, CtrlMask(controls, "CMULDIV")));
}
void QEngineCUDA::CDIV(const bitCapInt& toDiv, bitLenInt start, bitLenInt carryStart, bitLenInt length,
    const std::vector<bitLenInt>& controls)
{
    if (controls.empty()) {
        return DIV(toDiv, start, carryStart, length);
    }
    if (bi_compare_0(toDiv) == 0) {
        throw std::runtime_error("DIV by zero");
    }
    if (bi_compare_1(toDiv) == 0) {
        return;
    }
    Check(b200sv_muldiv(sv, 1, U64(toDiv), (int)start, (int)carryStart, (int)length, CtrlMask(controls, "CMULDIV")));
}

// ModNOut family: arithmetic.cpp:634-667, 737-775
void QEngineCUDA::MULModNOut(const bitCapInt& toMod, const bitCapInt& modN, bitLenInt inStart, bitLenInt outStart, bitLenInt length)
{
    SetReg(outStart, length, ZERO_BCI);
    if (bi_compare_0(toMod) == 0) {
        return;
    }
    Check(b200sv_modnout(sv, 0, U64(toMod), U64(modN), (int)inStart, (int)outStart, (int)length, 0U));
}
void QEngineCUDA::IMULModNOut(const bitCapInt& toMod, const bitCapInt& modN, bitLenInt inStart, bitLenInt outStart, bitLenInt length)
{
    if (bi_compare_0(toMod) == 0) {
        return;
    }
    Check(b200sv_modnout(sv, 1, U64(toMod), U64(modN), (int)inStart, (int)outStart, (int)length, 0U));
}
void QEngineCUDA::POWModNOut(const bitCapInt& base, const bitCapInt& modN, bitLenInt inStart, bitLenInt outStart, bitLenInt length)
{
    if (bi_compare_1(base) == 0) {
        return SetReg(outStart, length, ONE_BCI);
    }
    Check(b200sv_modnout(sv, 2, U64(base), U64(modN), (int)inStart, (int)outStart, (int)length, 0U));
}
void QEngineCUDA::CMULModNOut(const bitCapInt& toMod, const bitCapInt& modN, bitLenInt inStart, bitLenInt outStart,
    bitLenInt length, const std::vector<bitLenInt>& controls)
{
    if (controls.empty()) {
        return MULModNOut(toMod, modN, inStart, outStart, length);
    }
    SetReg(outStart, length, ZERO_BCI);
    Check(b200sv_modnout(sv, 0, U64(toMod), U64(modN), (int)inStart, (int)outStart, (int)length, CtrlMask(controls, "ModNOut")));
}
void QEngineCUDA::CIMULModNOut(const bitCapInt& toMod, const bitCapInt& modN, bitLenInt inStart, bitLenInt outStart,
    bitLenInt length, const std::vector<bitLenInt>& controls)
{
    if (controls.empty()) {
        return IMULModNOut(toMod, modN, inStart, outStart, length);
    }
    Check(b200sv_modnout(sv, 1, U64(toMod), U64(modN), (int)inStart, (int)outStart, (int)length, CtrlMask(controls, "ModNOut")));
}
void QEngineCUDA::CPOWModNOut(const bitCapInt& base, const bitCapInt& modN, bitLenInt inStart, bitLenInt outStart,
    bitLenInt length, const std::vector<bitLenInt>& controls)
{
    if (controls.empty()) {
        return POWModNOut(base, modN, inStart, outStart, length);
    }
    Check(b200sv_modnout(sv, 2, U64(base), U64(modN), (int)inStart, (int)outStart, (int)length, CtrlMask(controls, "ModNOut")));
}

// Indexed loads / adds from a classical table: arithmetic.cpp:983-1444.  The carry is measured (and cleared) first.
bitCapInt QEngineCUDA::IndexedLDA(bitLenInt indexStart, bitLenInt indexLength, bitLenInt valueStart, bitLenInt valueLength,
    const unsigned char* values, bool resetValue)
{
    if (isBadBitRange(indexStart, indexLength, qubitCount)) {
        throw std::invalid_argument("QEngineCUDA::IndexedLDA range is out-of-bounds!");
    }
    if (isBadBitRange(valueStart, valueLength, qubitCount)) {
        throw std::invalid_argument("QEngineCUDA::IndexedLDA range is out-of-bounds!");
    }
    if (IsZeroAmplitude()) {
        return ZERO_BCI;
    }
    if (resetValue) {
        SetReg(valueStart, valueLength, ZERO_BCI);
    }
    Check(b200sv_indexed(sv, 0, (int)indexStart, (int)indexLength, (int)valueStart, (int)valueLength, -1, 0, values));
    return ZERO_BCI;
}
bitCapInt QEngineCUDA::IndexedADC(bitLenInt indexStart, bitLenInt indexLength, bitLenInt valueStart, bitLenInt valueLength,
    bitLenInt carryIndex, const unsigned char* values)
{
    if (isBadBitRange(indexStart, indexLength, qubitCount) || isBadBitRange(valueStart, valueLength, qubitCount)) {
        throw std::invalid_argument("QEngineCUDA::IndexedADC range is out-of-bounds!");
    }
    if (carryIndex >= qubitCount) {
        throw std::invalid_argument("QEngineCUDA::IndexedADC carryIndex is out-of-bounds!");
    }
    if (IsZeroAmplitude()) {
        return ZERO_BCI;
    }
    int carryIn = 0;
    if (M(carryIndex)) {
        carryIn = 1;
        X(carryIndex);
    }
    Check(b200sv_indexed(sv, 1, (int)indexStart, (int)indexLength, (int)valueStart, (int)valueLength, (int)carryIndex, carryIn, values));
    return ZERO_BCI;
}
bitCapInt QEngineCUDA::IndexedSBC(bitLenInt indexStart, bitLenInt indexLength, bitLenInt valueStart, bitLenInt valueLength,
    bitLenInt carryIndex, const unsigned char* values)
{
    if (isBadBitRange(indexStart, indexLength, qubitCount) || isBadBitRange(valueStart, valueLength, qubitCount)) {
        throw std::invalid_argument("QEngineCUDA::IndexedSBC range is out-of-bounds!");
    }
    if (carryIndex >= qubitCount) {
        throw std::invalid_argument("QEngineCUDA::IndexedSBC carryIndex is out-of-bounds!");
    }
    if (IsZeroAmplitude()) {
        return ZERO_BCI;
    }
    int carryIn = 1;
    if (M(carryIndex)) {
        carryIn = 0;
        X(carryIndex);
    }
    Check(b200sv_indexed(sv, 2, (int)indexStart, (int)indexLength, (int)valueStart, (int)valueLength, (int)carryIndex, carryIn, values));
    return ZERO_BCI;
}
void QEngineCUDA::Hash(bitLenInt start, bitLenInt length, const unsigned char* values)
{
    Check(b200sv_hash(sv, (int)start, (int)length, values));
}
#undef U64
#endif

} // namespace Qrack
