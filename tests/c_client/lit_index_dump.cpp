// Host build of the v2 engine's literal prior order (dv_common.cuh: lit_index_hi / lit_index_lo), for
// tests/test_lit_index.py: writes to stdout, as little-endian u32, index(which, index_c, index_b) for the high table, then
// the low table, each in the order which, index_c, index_b (3 x 256 x 256 values per table).
#include <cstdio>
#include <vector>

#include "dv_common.cuh"

int main() {
    std::vector<uint32_t> out;
    out.reserve(2 * 3 * 256 * 256);
    for (int table = 0; table < 2; table++)
        for (uint32_t which = 0; which < 3; which++)
            for (uint32_t c = 0; c < 256; c++)
                for (uint32_t b = 0; b < 256; b++)
                    out.push_back(table == 0 ? dv::lit_index_hi(which, c, b) : dv::lit_index_lo(which, c, b));
    return fwrite(out.data(), sizeof(uint32_t), out.size(), stdout) == out.size() ? 0 : 1;
}
