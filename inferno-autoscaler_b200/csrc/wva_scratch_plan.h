// wva_scratch_plan.h — chunks of a materialised-path list (host only, no CUDA types).
//
// Each item of the list re-runs its chain with p[] in a scratch row of its own; item i needs len[i] doubles.  A chunk
// is the longest run of items from i0 on whose rows fit the capacity together; the rows are laid out back to back in
// list order.
#pragma once
#include <algorithm>
#include <cstddef>
#include <vector>

namespace wva {

struct ScratchChunk {
    size_t end = 0;           // the chunk is [i0, end); end == i0: item i0 alone does not fit
    long long doubles = 0;    // scratch the chunk needs
};

// The capacity of every materialised list: half the free device memory, or the scratch already held when that is more
// (memory a call already holds is missing from the free memory it reads).
inline long long scratch_cap_doubles(size_t freeBytes, size_t heldBytes) {
    return (long long)(std::max(freeBytes / 2, heldBytes) / 8);
}

// offs[k] = offset in doubles of item i0 + k's row (offs is resized to the chunk's length)
inline ScratchChunk scratch_chunk(const std::vector<long long>& len, size_t i0, long long capDoubles, std::vector<long long>& offs) {
    ScratchChunk c;
    offs.clear();
    for (c.end = i0; c.end < len.size() && c.doubles + len[c.end] <= capDoubles; ++c.end) {
        offs.push_back(c.doubles);
        c.doubles += len[c.end];
    }
    return c;
}

// The same chunk for a list of n items whose rows all have rowDoubles doubles: item i0 + k's row starts at k * rowDoubles.
inline ScratchChunk scratch_chunk_rows(size_t n, size_t i0, long long rowDoubles, long long capDoubles) {
    ScratchChunk c;
    c.end = i0 + std::min(n - i0, (size_t)(capDoubles / rowDoubles));
    c.doubles = (long long)(c.end - i0) * rowDoubles;
    return c;
}

}  // namespace wva
