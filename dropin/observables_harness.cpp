// observables_harness.cpp — replays a qscript circuit of U / CNOT gates followed by the observable queries of QInterface on a
// QEngine built by the reference's factory, and prints one result line per query in the qscript result format
// ("<op> <value> ..", as qrack_b200/qscript.py appends them).  Compiled against the reference's own QEngineCPU it produces the
// expected values of tests/golden/ref_observables_12q.*.npz (tests/golden/make_observables.py); compiled by dropin/Makefile
// against the drop-in, `--engine cuda` runs the same queries through QEngineCUDA's overrides.
//
//   observables_harness <script> [--engine cpu|cuda] [--dump FILE]
//
// Ops (tokens as in qrack_b200/qscript.py; <cs> = count then qubits):
//   qubits N | U q theta phi lambda | CNOT c t
//   ExpectationBitsAll|VarianceBitsAll <cs> offset
//   ExpectationBitsFactorized|VarianceBitsFactorized <cs> offset perm0 .. perm{2n-1}
//   ExpectationFloatsFactorized|VarianceFloatsFactorized <cs> weight0 .. weight{2n-1}
//   ExpectationPauliAll|VariancePauliAll <cs> pauli0 .. pauli{n-1}
//   ExpectationUnitaryAll|VarianceUnitaryAll <cs> theta0 phi0 lambda0 .. [eigenvalue0 .. eigenvalue{2n-1}]
//   ExpectationMatrixAll|VarianceMatrixAll <cs> <8 doubles per qubit: m00, m01, m10, m11 as re, im> [eigenvalues]
//                                         (the matrix form of ExpectationUnitaryAll / VarianceUnitaryAll)
//   GetReducedDensityMatrix <cs>          (prints the 2 4^n values of rho row-major, interleaved re / im)
//   HighestProbAllN n                     (prints the n most probable basis states, QInterface::HighestProbAll(n))
//   LossySave path p b | LossyLoad path  (LossySaveStateVector / LossyLoadStateVector)
#include "qfactory.hpp"

#include <algorithm>
#include <cstdio>
#include <memory>
#include <cstdlib>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>

using namespace Qrack;

int main(int argc, char** argv)
{
    if (argc < 2) {
        fprintf(stderr, "usage: %s <script> [--engine cpu|cuda] [--dump FILE]\n", argv[0]);
        return 2;
    }
    std::string engine = "cpu", dump;
    for (int a = 2; a + 1 < argc; a += 2) {
        const std::string s = argv[a];
        if (s == "--engine") {
            engine = argv[a + 1];
        } else if (s == "--dump") {
            dump = argv[a + 1];
        }
    }
    std::ifstream in(argv[1]);
    if (!in) {
        fprintf(stderr, "cannot open %s\n", argv[1]);
        return 2;
    }
    QInterfacePtr q;
    std::string line;
    while (std::getline(in, line)) {
        const size_t h = line.find('#');
        if (h != std::string::npos) {
            line.resize(h);
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
            q = CreateQuantumInterface((engine == "cuda") ? QINTERFACE_CUDA : QINTERFACE_CPU, (bitLenInt)n, ZERO_BCI, rng,
                ONE_CMPLX, false, false, false, -1, false);
            continue;
        }
        if (op == "U") {
            int t;
            double th, ph, la;
            ts >> t >> th >> ph >> la;
            q->U((bitLenInt)t, (real1_f)th, (real1_f)ph, (real1_f)la);
            continue;
        }
        if (op == "CNOT") {
            int c, t;
            ts >> c >> t;
            q->CNOT((bitLenInt)c, (bitLenInt)t);
            continue;
        }
        if (op == "LossySave") {
            std::string f;
            int p, b;
            ts >> f >> p >> b;
            q->LossySaveStateVector(f, p, b);
            continue;
        }
        if (op == "LossyLoad") {
            std::string f;
            ts >> f;
            q->LossyLoadStateVector(f);
            continue;
        }
        if (op == "HighestProbAllN") {
            size_t n;
            ts >> n;
            printf("%s", op.c_str());
            for (const bitCapInt& p : q->HighestProbAll(n)) {
                printf(" %llu", (unsigned long long)(bitCapIntOcl)p);
            }
            printf("\n");
            continue;
        }
        int k;
        ts >> k;
        std::vector<bitLenInt> bits(k);
        for (int i = 0; i < k; ++i) {
            int b;
            ts >> b;
            bits[i] = (bitLenInt)b;
        }
        if (op == "GetReducedDensityMatrix") {
            const size_t dim = (size_t)1U << k;
            std::vector<complex> rho(dim * dim);
            q->GetReducedDensityMatrix(bits, rho.data());
            printf("%s", op.c_str());
            for (const complex& z : rho) {
                printf(" %.17g %.17g", (double)real(z), (double)imag(z));
            }
            printf("\n");
            continue;
        }
        double r;
        if (op == "ExpectationBitsAll" || op == "VarianceBitsAll") {
            unsigned long long off;
            ts >> off;
            r = (op[0] == 'E') ? q->ExpectationBitsAll(bits, bitCapInt((uint64_t)off))
                               : q->VarianceBitsAll(bits, bitCapInt((uint64_t)off));
        } else if (op == "ExpectationBitsFactorized" || op == "VarianceBitsFactorized") {
            unsigned long long off, v;
            ts >> off;
            std::vector<bitCapInt> perms;
            while (ts >> v) {
                perms.push_back(bitCapInt((uint64_t)v));
            }
            r = (op[0] == 'E') ? q->ExpectationBitsFactorized(bits, perms, bitCapInt((uint64_t)off))
                               : q->VarianceBitsFactorized(bits, perms, bitCapInt((uint64_t)off));
        } else if (op == "ExpectationFloatsFactorized" || op == "VarianceFloatsFactorized" || op == "ExpectationUnitaryAll" ||
            op == "VarianceUnitaryAll") {
            double v;
            std::vector<real1_f> w;
            while (ts >> v) {
                w.push_back((real1_f)v);
            }
            if (op == "ExpectationFloatsFactorized") {
                r = q->ExpectationFloatsFactorized(bits, w);
            } else if (op == "VarianceFloatsFactorized") {
                r = q->VarianceFloatsFactorized(bits, w);
            } else {
                // past the 3 angles per qubit: the eigenvalues
                const size_t na = std::min(w.size(), 3U * bits.size());
                const std::vector<real1_f> angles(w.begin(), w.begin() + na), eig(w.begin() + na, w.end());
                r = (op[0] == 'E') ? q->ExpectationUnitaryAll(bits, angles, eig) : q->VarianceUnitaryAll(bits, angles, eig);
            }
        } else if (op == "ExpectationMatrixAll" || op == "VarianceMatrixAll") {
            std::vector<std::shared_ptr<complex>> mats;
            for (int i = 0; i < k; ++i) {
                std::shared_ptr<complex> m(new complex[4U], std::default_delete<complex[]>());
                for (int e = 0; e < 4; ++e) {
                    double re, im;
                    ts >> re >> im;
                    m.get()[e] = complex((real1)re, (real1)im);
                }
                mats.push_back(m);
            }
            double v;
            std::vector<real1_f> eig;
            while (ts >> v) {
                eig.push_back((real1_f)v);
            }
            r = (op[0] == 'E') ? q->ExpectationUnitaryAll(bits, mats, eig) : q->VarianceUnitaryAll(bits, mats, eig);
        } else if (op == "ExpectationPauliAll" || op == "VariancePauliAll") {
            int v;
            std::vector<Pauli> ps;
            while (ts >> v) {
                ps.push_back((Pauli)v);
            }
            r = (op[0] == 'E') ? q->ExpectationPauliAll(bits, ps) : q->VariancePauliAll(bits, ps);
        } else {
            fprintf(stderr, "unknown op '%s'\n", op.c_str());
            return 2;
        }
        printf("%s %.17g\n", op.c_str(), r);
    }
    if (!dump.empty() && q) {
        std::vector<complex> st((size_t)(bitCapIntOcl)q->GetMaxQPower());
        q->GetQuantumState(st.data());
        std::ofstream out(dump, std::ios::binary);
        out.write((const char*)st.data(), st.size() * sizeof(complex));
    }
    return 0;
}
