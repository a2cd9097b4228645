// TEST INFRASTRUCTURE (oracle/) — NOT product code.  std::sort of the C++ standard library this is compiled with, the call
// cloudProcessing makes on its points (src/cloudProcessing.cpp:181,236,306,345,416,455,525): the permutation it leaves, the order
// of equal keys included, for the three key types the handlers compare (double relative_time / robosense timestamp, float
// velodyne time, uint32 ouster t).  Built by oracle/cloud_processing.mk; tests/test_cloud_processing_pin.py pins the introsort
// restatement of tests/cloud_processing_ref.py against it.
#include <algorithm>
#include <cstdint>
#include <vector>

namespace {
template <class K> struct Rec {
    K key;
    std::int32_t idx;
};
template <class K> void sort_perm(const K* keys, std::int64_t n, std::int32_t* perm) {
    std::vector<Rec<K>> v(n);
    for (std::int64_t i = 0; i < n; ++i) v[i] = {keys[i], static_cast<std::int32_t>(i)};
    std::sort(v.begin(), v.end(), [](const Rec<K>& a, const Rec<K>& b) { return a.key < b.key; });
    for (std::int64_t i = 0; i < n; ++i) perm[i] = v[i].idx;
}
}  // namespace

extern "C" {
// perm[p] = the input index of the element std::sort leaves at position p
void srl_sort_perm_f64(const double* keys, std::int64_t n, std::int32_t* perm) { sort_perm(keys, n, perm); }
void srl_sort_perm_f32(const float* keys, std::int64_t n, std::int32_t* perm) { sort_perm(keys, n, perm); }
void srl_sort_perm_u32(const std::uint32_t* keys, std::int64_t n, std::int32_t* perm) { sort_perm(keys, n, perm); }
}
