// transform_emu.cpp -- the selection transform of selection.cu compiled for the CPU on top of tests/kernel_emu: transform_selection_kernel
// and the host's float64 matrices (edit_transform_matrices), exactly as libgsr runs them.  TEST INFRASTRUCTURE: built by
// tests/transform_reference.py.
#include "../kernel_emu/kernel_emu.cpp"

inline unsigned atomicOr(unsigned *p, unsigned v) { const unsigned o = *p; *p = o | v; return o; }   // blocks run one at a time
#include "../../godotgaussiansplatting_b200/csrc/selection.cu"

namespace {
struct TransformLaunch { gsr::TransformArgs a; };
template <int B, bool HALF>
void transform_body(void *p) { gsr::transform_selection_kernel<B, HALF>(static_cast<TransformLaunch *>(p)->a); }
void (*pick_transform(int bands, bool half))(void *) {
    switch (bands * 2 + (half ? 1 : 0)) {
        case 2: return &transform_body<1, false>;
        case 3: return &transform_body<1, true>;
        case 4: return &transform_body<2, false>;
        case 5: return &transform_body<2, true>;
        case 6: return &transform_body<3, false>;
        case 7: return &transform_body<3, true>;
        case 8: return &transform_body<4, false>;
        case 9: return &transform_body<4, true>;
        default: return nullptr;
    }
}
}  // namespace

// The 95 floats of gsr_transform_selection (GSR_BUF_EDIT_TRANSFORM) for to_source; GSR_ERR_INVALID for a singular L.
extern "C" int emu_edit_matrices(const float *to_source, float *out95) { return gsr::edit_transform_matrices(to_source, out95); }

// The library's float64 steps: Q = polar factor of L (row-major 3x3 in and out), M_l(Q) row-major.
extern "C" void emu_polar(const double *L9, double *Q9) {
    double L[3][3], Q[3][3];
    memcpy(L, L9, sizeof L);
    gsr::polar_factor(L, Q);
    memcpy(Q9, Q, sizeof Q);
}
extern "C" void emu_band_matrix(const double *Q9, int l, double *M) {
    double Q[3][3];
    memcpy(Q, Q9, sizeof Q);
    gsr::band_matrix(Q, l, M);
}

// transform_selection_kernel<bands, half> over every word: dst / src the store and its source (planes x plane_stride float4 each).
extern "C" int emu_transform_selection(int bands, int half, void *dst, const void *src, unsigned long long plane_stride, const uint32_t *selected,
                                       unsigned words, const float *m95) {
    TransformLaunch l;
    memset(&l, 0, sizeof l);
    l.a.dst = static_cast<float4 *>(dst); l.a.src = static_cast<const float4 *>(src); l.a.plane_stride = plane_stride;
    l.a.selected = selected; l.a.words = words;
    memcpy(l.a.m, m95, sizeof l.a.m);
    void (*body)(void *) = pick_transform(bands, half != 0);
    if (!body) return -1;
    const unsigned blocks = (words + 7u) / 8u;
    if (blocks) run_blocks(blocks, 256u, body, &l);
    return 0;
}
