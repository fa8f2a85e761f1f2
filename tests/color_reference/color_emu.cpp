// color_emu.cpp -- the selection colour edit of selection.cu compiled for the CPU on top of tests/kernel_emu: recolor_selection_kernel and
// the host's float64 constants (edit_color_constants), exactly as libgsr runs them.  TEST INFRASTRUCTURE: built by tests/color_reference.py.
#include "../kernel_emu/kernel_emu.cpp"

inline unsigned atomicOr(unsigned *p, unsigned v) { const unsigned o = *p; *p = o | v; return o; }   // blocks run one at a time
#include "../../godotgaussiansplatting_b200/csrc/selection.cu"

namespace {
struct RecolorLaunch { gsr::RecolorArgs a; };
template <int B, bool HALF>
void recolor_body(void *p) { gsr::recolor_selection_kernel<B, HALF>(static_cast<RecolorLaunch *>(p)->a); }
void (*pick_recolor(int bands, bool half))(void *) {
    switch (bands * 2 + (half ? 1 : 0)) {
        case 2: return &recolor_body<1, false>;
        case 3: return &recolor_body<1, true>;
        case 4: return &recolor_body<2, false>;
        case 5: return &recolor_body<2, true>;
        case 6: return &recolor_body<3, false>;
        case 7: return &recolor_body<3, true>;
        case 8: return &recolor_body<4, false>;
        case 9: return &recolor_body<4, true>;
        default: return nullptr;
    }
}
}  // namespace

// The 41 floats of gsr_recolor_selection (GSR_BUF_EDIT_COLOR) for a gsr_color_edit.
extern "C" void emu_color_constants(const gsr_color_edit *edit, float *out41) { gsr::edit_color_constants(edit, out41); }

// recolor_selection_kernel<bands, half> over every word: dst / src the store and its source (planes x plane_stride float4 each; the same
// pointer for an edit in place).
extern "C" int emu_recolor_selection(int bands, int half, void *dst, const void *src, unsigned long long plane_stride, const uint32_t *selected,
                                     unsigned words, const float *k41) {
    RecolorLaunch l;
    memset(&l, 0, sizeof l);
    l.a.dst = static_cast<float4 *>(dst); l.a.src = static_cast<const float4 *>(src); l.a.plane_stride = plane_stride;
    l.a.selected = selected; l.a.words = words;
    memcpy(l.a.k, k41, sizeof l.a.k);
    void (*body)(void *) = pick_recolor(bands, half != 0);
    if (!body) return -1;
    const unsigned blocks = (words + 7u) / 8u;
    if (blocks) run_blocks(blocks, 256u, body, &l);
    return 0;
}
