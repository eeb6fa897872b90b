// dropin/gates_harness.cpp — TEST INFRASTRUCTURE, not product code.
//
// Replays the qscript ops of the two-target, parity-rotation and uniformly controlled gate fixtures (qrack_b200/qscript.py
// grammar) through the public API of whatever libqrack it is linked against, and dumps the final state vector.
// tests/golden/make_gates.py links it against the reference's own QEngineCPU (oracle/_ref/f{32,64}/libqrack.a) to write
// tests/golden/ref_gates_9q.f{32,64}.npz.
//
//   gates_harness <script> --dump FILE
//
// Ops: qubits N, H q, X q, U q theta phi lambda, CNOT c t, XMask mask, ISwap|SqrtSwap a b, FSim theta phi a b,
// CSwap|AntiCSwap <cs> a b, UniformParityRZ mask angle, CUniformParityRZ <cs> mask angle,
// UniformlyControlledSingleBit <cs> t <ss> skipValueMask <m8 per table entry>, UniformlyControlledRY|RZ <cs> t angles.
#include "qfactory.hpp"
#include "qparity.hpp"

#include <cstdio>
#include <fstream>
#include <memory>
#include <sstream>
#include <string>
#include <vector>

using namespace Qrack;

static std::vector<bitLenInt> read_bits(std::istringstream& ts)
{
    int k;
    ts >> k;
    std::vector<bitLenInt> bits(k);
    for (int i = 0; i < k; ++i) {
        int b;
        ts >> b;
        bits[i] = (bitLenInt)b;
    }
    return bits;
}

int main(int argc, char** argv)
{
    if (argc != 4 || std::string(argv[2]) != "--dump") {
        fprintf(stderr, "usage: %s <script> --dump FILE\n", argv[0]);
        return 2;
    }
    std::ifstream in(argv[1]);
    QInterfacePtr q;
    std::string line;
    while (std::getline(in, line)) {
        const size_t h = line.find('#');
        if (h != std::string::npos) {
            line = line.substr(0, h);
        }
        std::istringstream ts(line);
        std::string op;
        if (!(ts >> op)) {
            continue;
        }
        if (op == "qubits") {
            int n;
            ts >> n;
            qrack_rand_gen_ptr rng = std::make_shared<qrack_rand_gen>();
            rng->seed(20250921U);
            q = CreateQuantumInterface(QINTERFACE_CPU, (bitLenInt)n, ZERO_BCI, rng, ONE_CMPLX, false, false, false, -1, false);
        } else if (op == "H" || op == "X") {
            int t;
            ts >> t;
            (op == "H") ? q->H((bitLenInt)t) : q->X((bitLenInt)t);
        } else if (op == "U") {
            int t;
            double th, ph, la;
            ts >> t >> th >> ph >> la;
            q->U((bitLenInt)t, (real1_f)th, (real1_f)ph, (real1_f)la);
        } else if (op == "CNOT" || op == "ISwap" || op == "SqrtSwap") {
            int a, b;
            ts >> a >> b;
            if (op == "CNOT") {
                q->CNOT((bitLenInt)a, (bitLenInt)b);
            } else if (op == "ISwap") {
                q->ISwap((bitLenInt)a, (bitLenInt)b);
            } else {
                q->SqrtSwap((bitLenInt)a, (bitLenInt)b);
            }
        } else if (op == "XMask") {
            unsigned long long m;
            ts >> m;
            q->XMask(bitCapInt(m));
        } else if (op == "FSim") {
            double th, ph;
            int a, b;
            ts >> th >> ph >> a >> b;
            q->FSim((real1_f)th, (real1_f)ph, (bitLenInt)a, (bitLenInt)b);
        } else if (op == "CSwap" || op == "AntiCSwap") {
            const std::vector<bitLenInt> c = read_bits(ts);
            int a, b;
            ts >> a >> b;
            (op == "CSwap") ? q->CSwap(c, (bitLenInt)a, (bitLenInt)b) : q->AntiCSwap(c, (bitLenInt)a, (bitLenInt)b);
        } else if (op == "UniformParityRZ" || op == "CUniformParityRZ") {
            std::vector<bitLenInt> c;
            if (op[0] == 'C') {
                c = read_bits(ts);
            }
            unsigned long long m;
            double a;
            ts >> m >> a;
            std::shared_ptr<QParity> qp = std::dynamic_pointer_cast<QParity>(q);
            (op[0] == 'C') ? qp->CUniformParityRZ(c, bitCapInt(m), (real1_f)a) : qp->UniformParityRZ(bitCapInt(m), (real1_f)a);
        } else if (op == "UniformlyControlledSingleBit") {
            const std::vector<bitLenInt> c = read_bits(ts);
            int t, ns;
            ts >> t >> ns;
            std::vector<bitCapInt> skips(ns);
            for (int i = 0; i < ns; ++i) {
                unsigned long long p;
                ts >> p;
                skips[i] = bitCapInt(p);
            }
            unsigned long long svm;
            ts >> svm;
            std::vector<complex> m((size_t)4U << (c.size() + ns));
            for (complex& z : m) {
                double re, im;
                ts >> re >> im;
                z = complex((real1)re, (real1)im);
            }
            q->UniformlyControlledSingleBit(c, (bitLenInt)t, m.data(), skips, bitCapInt(svm));
        } else if (op == "UniformlyControlledRY" || op == "UniformlyControlledRZ") {
            const std::vector<bitLenInt> c = read_bits(ts);
            int t;
            ts >> t;
            std::vector<real1> angles((size_t)1U << c.size());
            for (real1& a : angles) {
                double v;
                ts >> v;
                a = (real1)v;
            }
            (op == "UniformlyControlledRY") ? q->UniformlyControlledRY(c, (bitLenInt)t, angles.data())
                                            : q->UniformlyControlledRZ(c, (bitLenInt)t, angles.data());
        } else {
            fprintf(stderr, "unknown op '%s'\n", op.c_str());
            return 2;
        }
    }
    std::vector<complex> st((size_t)(bitCapIntOcl)q->GetMaxQPower());
    q->GetQuantumState(st.data());
    std::ofstream out(argv[3], std::ios::binary);
    out.write((const char*)st.data(), st.size() * sizeof(complex));
    return 0;
}
