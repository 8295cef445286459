// tests/emu/emu_merkle.cpp -- TEST INFRASTRUCTURE: the CPU emulation of emu.cpp (included whole, so a launch of
// k_merkle_chunk is the same emulated CTA code) plus batched Merkle trees: the library's batch loop and per-tree
// views (fri_merkle.cuh: merkle_batch_launches, merkle_view) over emulated launches.
// It is NOT a fallback: nothing in the product loads this library.
//
// Build: g++ -O2 -std=c++17 -shared -fPIC -o libsa_emu_merkle.so emu_merkle.cpp
#include "emu.cpp"

extern "C" {

// sa_merkle_tree_batch: every launch runs the CTAs of each tree of its group, and a tree's first launch from its
// codeword zeroes node 0 as CTA 0 of k_merkle_chunk does (the trees do not meet: without arrival counters there is
// no fused top, which the GPU tests check)
int emu_merkle_tree_batch(uint8_t *trees, const uint64_t *values, size_t n, size_t batch) {
    MerkleArgs a;
    memset(&a, 0, sizeof(a));
    a.tree = (uint64_t *)trees;
    a.tree_stride = 16 * (long long)n;
    a.row_stride = (long long)n;
    a.width = (long long)n;
    a.mode = 1;
    a.values = (const fe *)values;
    return merkle_batch_launches(
        a, (long long)batch, [](int) { return (unsigned int *)nullptr; }, g_mk_shape.c_str(),
        [](MerkleArgs &m, int trees, bool) {
            for (int b = 0; b < trees; b++) {
                const MerkleArgs v = merkle_view(m, b);
                if (v.mode == 1) memset(v.tree, 0, 64);
                emu_merkle_chunk(v);
            }
            return 0;
        });
}

}  // extern "C"
