// compressed_emu.cpp -- the compressed PLY kernels compiled for the CPU on top of tests/kernel_emu: compress_bounds_kernel,
// compress_key_kernel, the library's Onesweep pair sort (kernel_emu's emu_sort_pairs) and compress_chunk_kernel of compressed_ply.cu, in
// the order gsr_export_compressed_ply launches them, and compressed_to_soa_kernel of ingest.cu as gsr_upload_compressed_ply launches it.
// TEST INFRASTRUCTURE: built by tests/compressed_reference.py.
#include "../kernel_emu/kernel_emu.cpp"

// fibers of one thread: sequential
inline unsigned atomicMin(unsigned *p, unsigned v) { const unsigned o = *p; *p = o < v ? o : v; return o; }
inline unsigned atomicMax(unsigned *p, unsigned v) { const unsigned o = *p; *p = o > v ? o : v; return o; }
#include "../../godotgaussiansplatting_b200/csrc/compressed_ply.cu"

namespace {
template <int B, bool HALF>
void chunk_body(void *p) { gsr::compress_chunk_kernel<B, HALF>(*static_cast<gsr::CompressArgs *>(p)); }
template <int B, bool HALF>
void decode_body(void *p) { gsr::compressed_to_soa_kernel<B, HALF>(*static_cast<gsr::DecompressArgs *>(p)); }
void (*pick_chunk(int bands, bool half))(void *) {
    switch (bands * 2 + (half ? 1 : 0)) {
        case 2: return &chunk_body<1, false>;
        case 3: return &chunk_body<1, true>;
        case 4: return &chunk_body<2, false>;
        case 5: return &chunk_body<2, true>;
        case 6: return &chunk_body<3, false>;
        case 7: return &chunk_body<3, true>;
        case 8: return &chunk_body<4, false>;
        case 9: return &chunk_body<4, true>;
        default: return nullptr;
    }
}
void (*pick_decode(int bands, bool half))(void *) {
    switch (bands * 2 + (half ? 1 : 0)) {
        case 2: return &decode_body<1, false>;
        case 3: return &decode_body<1, true>;
        case 4: return &decode_body<2, false>;
        case 5: return &decode_body<2, true>;
        case 6: return &decode_body<3, false>;
        case 7: return &decode_body<3, true>;
        case 8: return &decode_body<4, false>;
        case 9: return &decode_body<4, true>;
        default: return nullptr;
    }
}
}  // namespace

// gsr_export_compressed_ply's kernels on a host store (planes x plane_stride float4) and masks (hidden == NULL: not in use).  Returns the
// exported count.  With chunks / packed / sh and a count that fits cap_rows, the key pass, the sort and the chunk pass then fill them;
// keys_out (n entries, nullable) receives the key pass's keys before the sort and vals_out (n, nullable) the sorted slots.
// -1: bad arguments.
extern "C" long long emu_compress(int bands, int half, const void *soa, unsigned long long plane_stride, unsigned long long n,
                                  const uint32_t *hidden, const uint32_t *selected, int selected_only, int morton, int degree, uint32_t *keys_out,
                                  uint32_t *vals_out, float *chunks, uint32_t *packed, uint8_t *sh, unsigned long long cap_rows) {
    void (*body)(void *) = pick_chunk(bands, half != 0);
    if (!body || degree < 0 || degree > bands - 1) return -1;
    if (n == 0 || (selected_only && !hidden)) return 0;
    gsr::CompressArgs a;
    memset(&a, 0, sizeof a);
    a.soa = static_cast<const float4 *>(soa); a.plane_stride = plane_stride; a.n = n;
    a.hidden = hidden; a.selected = selected; a.selected_only = selected_only ? 1u : 0u; a.morton = morton ? 1u : 0u; a.degree = degree;
    gsr::CompressBounds b;
    for (int k = 0; k < 3; ++k) { b.lo[k] = 0xFFFFFFFFu; b.hi[k] = 0u; }
    b.count = 0ull;
    a.bounds = &b;
    const unsigned long long warps = (n + 31ull) / 32ull, need = (warps + 7ull) / 8ull;
    run_blocks((unsigned)(need < 2048ull ? need : 2048ull), 256, [](void *p) { gsr::compress_bounds_kernel(*static_cast<gsr::CompressArgs *>(p)); }, &a);
    const unsigned long long count = b.count;
    if (!chunks || !packed || count > cap_rows || count == 0) return (long long)count;
    std::vector<uint32_t> keys(n), vals(n);
    uint32_t sort_n = 0u;
    a.keys = keys.data(); a.vals = vals.data(); a.sort_n = &sort_n;
    run_blocks((unsigned)((n + 255ull) / 256ull), 256, [](void *p) { gsr::compress_key_kernel(*static_cast<gsr::CompressArgs *>(p)); }, &a);
    if (sort_n != (uint32_t)n) return -1;
    if (keys_out) memcpy(keys_out, keys.data(), sizeof(uint32_t) * n);
    emu_sort_pairs(keys.data(), vals.data(), (uint32_t)n, (uint32_t)n, 2);
    if (vals_out) memcpy(vals_out, vals.data(), sizeof(uint32_t) * n);
    a.rows = count; a.chunks = chunks; a.packed = packed; a.sh = sh;
    run_blocks((unsigned)((count + 255ull) / 256ull), 256, body, &a);
    return (long long)count;
}

// gsr_upload_compressed_ply's kernel: rows [0, rows) into splats [first, first + rows) of a host store.  -1: bad arguments.
extern "C" int emu_decompress(int bands, int half, const float *chunks, const uint32_t *packed, const uint8_t *sh, unsigned long long rows,
                              unsigned chunk_floats, int degree, float creation_time, void *soa, unsigned long long plane_stride,
                              unsigned long long first) {
    void (*body)(void *) = pick_decode(bands, half != 0);
    if (!body || degree < 0 || degree > 3 || (chunk_floats != 12u && chunk_floats != 18u)) return -1;
    gsr::DecompressArgs a;
    memset(&a, 0, sizeof a);
    a.chunks = chunks; a.packed = packed; a.sh = sh; a.rows = rows; a.chunk_floats = chunk_floats; a.degree = degree;
    a.creation_time = creation_time; a.soa = static_cast<float4 *>(soa); a.plane_stride = plane_stride; a.first = first;
    if (rows) run_blocks((unsigned)((rows + 255ull) / 256ull), 256, body, &a);
    return 0;
}
