// TEST INFRASTRUCTURE (oracle/) — NOT product code.  std::shuffle of the C++ standard library this is compiled with, the call
// buildFrame makes (src/lioOptimization.cpp:838-847, boost::mt19937_64 = std::mt19937_64 as in shim/srl_shim_ext.h).  Built twice
// by oracle/build_frame.mk: as is (libstdc++ draws with Lemire's 128-bit multiply) and with -U__SIZEOF_INT128__ (libstdc++ takes its
// division downscale, the rule of libstdc++ <= 10).  tests/test_build_frame_model.py pins the numpy model against both.
#include <algorithm>
#include <cstdint>
#include <random>
#include <vector>

namespace {
// a uniform random bit generator that replays given 64-bit words
struct Replay {
    using result_type = std::uint64_t;
    const std::uint64_t* w;
    std::int64_t n, pos;
    static constexpr result_type min() { return 0; }
    static constexpr result_type max() { return ~std::uint64_t(0); }
    result_type operator()() { return pos < n ? w[pos++] : (++pos, 0); }
};
}  // namespace

extern "C" {

int32_t probe_int128(void) {
#ifdef __SIZEOF_INT128__
    return 1;
#else
    return 0;
#endif
}

// shuffles of sizes sizes[0..k) in a row with ONE default-seeded engine (buildFrame's two calls); perm_out: the concatenated
// permutations (element index that ends at each position); returns the engine's next output
uint64_t probe_shuffle_mt(const int64_t* sizes, int32_t k, int32_t* perm_out) {
    std::mt19937_64 g;
    for (int32_t s = 0; s < k; ++s) {
        std::vector<int32_t> a((size_t)sizes[s]);
        for (int64_t i = 0; i < sizes[s]; ++i) a[(size_t)i] = (int32_t)i;
        std::shuffle(a.begin(), a.end(), g);
        std::copy(a.begin(), a.end(), perm_out);
        perm_out += sizes[s];
    }
    return g();
}

// one shuffle of n over a replayed word stream; returns the words consumed (> n_words: the stream ran out)
int64_t probe_shuffle_replay(const uint64_t* words, int64_t n_words, int64_t n, int32_t* perm_out) {
    Replay g{words, n_words, 0};
    std::vector<int32_t> a((size_t)n);
    for (int64_t i = 0; i < n; ++i) a[(size_t)i] = (int32_t)i;
    std::shuffle(a.begin(), a.end(), g);
    std::copy(a.begin(), a.end(), perm_out);
    return g.pos;
}

}  // extern "C"
