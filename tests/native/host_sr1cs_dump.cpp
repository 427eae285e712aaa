// The C++ mirror's Sr1csAdapter (snark_b200/host/ark_relations.hpp) on an R1CS read from a file, for
// tests/test_sr1cs_oracle.py:  ./host_sr1cs_dump <curve 0|1> <file>
//
// Input (whitespace separated, field elements as 8 hex u32 words of the Montgomery form, low word first):
//   n_instance n_witness n_rows
//   z[1 .. n_instance + n_witness)                         (z[0] = ONE is implied)
//   n_rows x 3 lines: count, then count pairs (col, coeff)  (A_i, B_i, C_i)
// Output: the R1CS as to_matrices() holds it after finalize ("S k i" + (col, coeff) pairs per row), then the converted
// system ("N n_instance n_witness", "D j i" rows of its two arguments, "Z" one line per element of instance || witness).
// With a third argument "time": only "T <seconds of the conversion> <constraints>".
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <string>

#include "../../snark_b200/host/ark_snark.hpp"

using namespace ark_relations::gr1cs;
using ark_relations::sr1cs::Sr1csAdapter;

template <class F>
static F read_fr(std::istream& in) {
    F x = F::zero();
    for (int i = 0; i < F::N; i++) {
        std::string w;
        in >> w;
        x.v[i] = (uint32_t)strtoul(w.c_str(), nullptr, 16);
    }
    return x;
}

template <class F>
static void print_row(const char* tag, int k, size_t i, const std::vector<std::pair<F, size_t>>& row) {
    printf("%s %d %zu", tag, k, i);
    for (const auto& [c, col] : row) {
        printf(" %zu", col);
        for (int w = 0; w < F::N; w++) printf(" %08x", c.v[w]);
    }
    printf("\n");
}

template <class Curve>
static int run(const char* path, bool timing) {
    using F = typename Curve::Fr;
    std::ifstream in(path);
    size_t n_inst = 0, n_wit = 0, n_rows = 0;
    if (!(in >> n_inst >> n_wit >> n_rows) || n_inst == 0) return 2;
    auto cs = ConstraintSystemRef<F>::new_ref();
    std::vector<Variable> var{Variable::One()};
    for (size_t j = 1; j < n_inst; j++) {
        const F v = read_fr<F>(in);
        var.push_back(cs.new_input_variable([=] { return v; }));
    }
    for (size_t j = 0; j < n_wit; j++) {
        const F v = read_fr<F>(in);
        var.push_back(cs.new_witness_variable([=] { return v; }));
    }
    for (size_t i = 0; i < n_rows; i++) {
        LinearCombination<F> lcs[3];
        for (int k = 0; k < 3; k++) {
            size_t cnt = 0;
            in >> cnt;
            for (size_t t = 0; t < cnt; t++) {
                size_t col = 0;
                in >> col;
                const F c = read_fr<F>(in);
                lcs[k].terms.emplace_back(c, var.at(col));
            }
        }
        cs.enforce_r1cs_constraint([&] { return lcs[0]; }, [&] { return lcs[1]; }, [&] { return lcs[2]; });
    }
    if (!in) return 2;
    cs.finalize();
    const auto src = cs.to_matrices().at(R1CS_PREDICATE_LABEL);
    for (int k = 0; k < 3 && !timing; k++)
        for (size_t i = 0; i < src[k].size(); i++) print_row("S", k, i, src[k][i]);
    if (timing) {   // the conversion alone, for tools/sr1cs_probe.py
        const auto t0 = std::chrono::steady_clock::now();
        auto out = Sr1csAdapter<F>::r1cs_to_sr1cs_with_assignment(cs.inner());
        printf("T %.6f %zu\n", std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(), out.num_constraints());
        return 0;
    }
    auto out = Sr1csAdapter<F>::r1cs_to_sr1cs_with_assignment(cs.inner());
    printf("N %zu %zu\n", out.num_instance_variables(), out.num_witness_variables());
    const auto dst = out.to_matrices().at(SR1CS_PREDICATE_LABEL);
    for (int j = 0; j < 2; j++)
        for (size_t i = 0; i < dst[j].size(); i++) print_row("D", j, i, dst[j][i]);
    std::vector<F> z = out->instance_assignment();
    z.insert(z.end(), out->witness_assignment().begin(), out->witness_assignment().end());
    for (const F& v : z) {
        printf("Z");
        for (int w = 0; w < F::N; w++) printf(" %08x", v.v[w]);
        printf("\n");
    }
    return 0;
}

int main(int argc, char** argv) {
    if (argc != 3 && !(argc == 4 && strcmp(argv[3], "time") == 0)) {
        printf("usage: %s <curve 0|1> <file> [time]\n", argv[0]);
        return 64;
    }
    const bool timing = argc == 4;
    try {
        return atoi(argv[1]) == 0 ? run<b2s::Bls12_381>(argv[2], timing) : run<b2s::Bn254>(argv[2], timing);
    } catch (const std::exception& e) {
        printf("ERROR %s\n", e.what());
        return 2;
    }
}
