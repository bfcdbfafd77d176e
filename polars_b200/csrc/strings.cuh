// strings.cuh — the device string column and the string operators shared by strings.cu and string_rank.cu.
#pragma once
#include "common.cuh"

namespace plb {

// Arrow LargeBinary / LargeUtf8 on the device, rows concatenated from the caller's chunks (import_string).
struct DevStr {
    int64_t len = 0, data_bytes = 0, null_count = 0;
    DevPtr offsets;    // (len + 1) x int64, offsets[0] == 0
    DevPtr data;       // data_bytes, plus 16 bytes of padding that any kernel may read
    DevPtr validity;   // word-padded bitmap or null
    const int64_t* off() const { return as<int64_t>(offsets); }
    const uint8_t* bytes() const { return as<uint8_t>(data); }
    const uint32_t* vm() const { return validity ? as<uint32_t>(validity) : nullptr; }
};

DevStr import_string(const bl_string_column* chunks, int n_chunks);
// code[row] = first row holding the same bytes (UInt32, validity = the input's); *n_distinct = distinct non-null values
DevCol op_string_codes(const DevStr& s, int64_t* n_distinct);
// dense lexicographic rank (UInt32, 1-based, validity = the input's; descending: the largest value is 1)
DevCol op_string_rank(const DevStr& s, bool descending, int64_t* n_distinct);

}  // namespace plb
