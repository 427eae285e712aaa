// The C++ mirror's instance outlining (snark_b200/host/ark_relations.hpp: perform_instance_outlining, outline_r1cs,
// outline_sr1cs) on a constraint system read from a file, for tests/test_outline_oracle.py:
//   ./host_outline_dump <curve 0|1> <file> [time]
//
// Input (whitespace separated, field elements as 8 hex u32 words of the Montgomery form, low word first):
//   strategy n_instance n_witness n_constraints      strategy: 0 none, 1 outline_r1cs (label "R1CS"), 2 outline_sr1cs ("SR1CS")
//   z[1 .. n_instance + n_witness)                    (z[0] = ONE is implied)
//   per constraint: its label R or S, then per argument (3 or 2): count, then count triples (kind index coeff), kind 0 Zero,
//   1 One, 2 Instance, 3 Witness.  Each argument goes through the builder as that LinearCombination, uncompactified.
// Both predicates, "R1CS" and "SR1CS", are registered.  Output after finalize(): "N n_instance n_witness", every row of
// to_matrices() as "M <label> <argument> <row>" + (col, coeff) pairs in term order, and "Z" one line per element of
// instance || witness.  With "time": only "T <seconds of finalize()> <constraints>".
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <string>

#include "../../snark_b200/host/ark_snark.hpp"

using namespace ark_relations::gr1cs;

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

template <class Curve>
static int run(const char* path, bool timing) {
    using F = typename Curve::Fr;
    std::ifstream in(path);
    int strategy = 0;
    size_t n_inst = 0, n_wit = 0, n_cons = 0;
    if (!(in >> strategy >> n_inst >> n_wit >> n_cons) || n_inst == 0) return 2;
    auto cs = ConstraintSystemRef<F>::new_ref();
    cs->register_predicate(SR1CS_PREDICATE_LABEL, PredicateConstraintSystem<F>::new_sr1cs_predicate());
    for (size_t j = 1; j < n_inst; j++) {
        const F v = read_fr<F>(in);
        cs.new_input_variable([=] { return v; });
    }
    for (size_t j = 0; j < n_wit; j++) {
        const F v = read_fr<F>(in);
        cs.new_witness_variable([=] { return v; });
    }
    for (size_t i = 0; i < n_cons; i++) {
        std::string label;
        in >> label;
        const size_t arity = label == "R" ? 3 : 2;
        std::vector<LinearCombination<F>> lcs(arity);
        for (size_t k = 0; k < arity; k++) {
            size_t cnt = 0;
            in >> cnt;
            for (size_t t = 0; t < cnt; t++) {
                int kind = 0;
                size_t idx = 0;
                in >> kind >> idx;
                const F c = read_fr<F>(in);
                const Variable v = kind == 0 ? Variable::Zero() : kind == 1 ? Variable::One() : kind == 2 ? Variable::instance(idx) : Variable::witness(idx);
                lcs[k].terms.emplace_back(c, v);
            }
        }
        std::vector<typename ConstraintSystem<F>::LazyLc> lazy;
        for (size_t k = 0; k < arity; k++) lazy.push_back([&, k] { return lcs[k]; });
        cs.enforce_constraint(label == "R" ? R1CS_PREDICATE_LABEL : SR1CS_PREDICATE_LABEL, lazy);
    }
    if (!in) return 2;
    if (strategy == 1) cs->set_instance_outliner({R1CS_PREDICATE_LABEL, outline_r1cs<F>});
    if (strategy == 2) cs->set_instance_outliner({SR1CS_PREDICATE_LABEL, outline_sr1cs<F>});
    const auto t0 = std::chrono::steady_clock::now();
    cs->finalize();
    if (timing) {   // finalize() alone, for tools/outline_probe.py
        printf("T %.6f %zu\n", std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(), cs->num_constraints());
        return 0;
    }
    printf("N %zu %zu\n", cs->num_instance_variables(), cs->num_witness_variables());
    for (const auto& [label, mats] : cs->to_matrices())
        for (size_t k = 0; k < mats.size(); k++)
            for (size_t i = 0; i < mats[k].size(); i++) {
                printf("M %s %zu %zu", label.c_str(), k, i);
                for (const auto& [c, col] : mats[k][i]) {
                    printf(" %zu", col);
                    for (int w = 0; w < F::N; w++) printf(" %08x", c.v[w]);
                }
                printf("\n");
            }
    std::vector<F> z = cs->instance_assignment();
    z.insert(z.end(), cs->witness_assignment().begin(), cs->witness_assignment().end());
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
