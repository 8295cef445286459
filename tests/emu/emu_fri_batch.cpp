// tests/emu/emu_fri_batch.cpp -- TEST INFRASTRUCTURE: the CPU emulation of emu.cpp (included whole, so a launch of
// k_merkle_chunk is the same emulated CTA code) plus the batched FRI commit: the library's round schedule
// (fri_merkle.cuh: fri_commit_batch_rounds), its per-tree views of the fused fold + tree round (merkle_tree_args) and
// its launch groups (merkle_batch_launches) over emulated launches.
// It is NOT a fallback: nothing in the product loads this library.
//
// Build: g++ -O2 -std=c++17 -shared -fPIC -o libsa_emu_fri_batch.so emu_fri_batch.cpp
#include "emu.cpp"

namespace {

// what the library's ops do on the device, on the host: every tree of a launch group runs its CTAs (without arrival
// counters, so without the fused top), the roots are read from the trees, the tables and scalars stay host vectors
struct EmuFriOps {
    long long B;
    sa_fri_challenge_batch_fn fn;
    void *user;
    MerkleArgs last;  // the round's trees
    std::vector<fe> tab, s;
    int tree(const MerkleArgs &a, int) {
        last = a;
        return merkle_batch_launches(
            a, B, [](int) { return (unsigned int *)nullptr; }, g_mk_shape.c_str(), [](MerkleArgs &m, int trees, bool) {
                for (int b = 0; b < trees; b++) {
                    const MerkleArgs v = merkle_tree_args(m, b);
                    if (v.mode == 1) memset(v.tree, 0, 64);  // CTA 0 of a tree's first launch from its codeword
                    emu_merkle_chunk(v);
                }
                return 0;
            });
    }
    int roots(int, uint8_t *out) {
        for (long long b = 0; b < B; b++) memcpy(out + 64 * b, last.tree + b * last.tree_stride + 8, 64);
        return SA_OK;
    }
    int challenge(int r, const uint8_t *roots, uint64_t *alphas, int want) { return fn(user, r, roots, alphas, want); }
    int xinv(const fe **out, const fe &omega, long long len) {
        tab = pow_table(fe_mont_inv(fe_to_mont(omega)), len / 2, 0);
        *out = tab.data();
        return SA_OK;
    }
    int scalars(const fe **dev, int, const fe *host) {
        s.assign(host, host + B);
        *dev = s.data();
        return SA_OK;
    }
};

}  // namespace

extern "C" {

// sa_fri_commit_batch with host buffers: the library's checks, then its round schedule over emulated launches
int emu_fri_commit_batch(uint64_t *layers, uint8_t *trees, const uint64_t *codewords, size_t n, size_t batch,
                         int rounds, const uint64_t *offset, const uint64_t *omega,
                         sa_fri_challenge_batch_fn challenge, void *user) {
    SA_TRY(fri_commit_batch_check(layers, trees, codewords, n, batch, rounds, offset, omega, (const void *)challenge));
    if (batch == 0) return SA_OK;
    EmuFriOps ops{(long long)batch, challenge, user, MerkleArgs(), {}, {}};
    return fri_commit_batch_rounds(ops, (fe *)layers, (uint64_t *)trees, (const fe *)codewords, (long long)n,
                                   (long long)batch, rounds, fe_from_limbs(offset), fe_from_limbs(omega));
}

}  // extern "C"
