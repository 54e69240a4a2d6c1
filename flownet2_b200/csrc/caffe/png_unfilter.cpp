// PNG's per-row filters undone on the host (include/fn2_flow.h, fn2_png_unfilter).  Paeth and Average depend on the bytes
// just reconstructed to their left, so a row is sequential; flownet2_b200.kitti runs one call per file on its reader pool
// (ctypes releases the GIL for the call).
#include <cstdint>
#include <cstdlib>
#include <cstring>

#include "../../../include/fn2_flow.h"

namespace fn2 { void set_error(const char* fmt, ...); }

static inline uint8_t paeth(int a, int b, int c) {
    const int p = a + b - c, pa = std::abs(p - a), pb = std::abs(p - b), pc = std::abs(p - c);
    return (uint8_t)(pa <= pb && pa <= pc ? a : pb <= pc ? b : c);
}

extern "C" int fn2_png_unfilter(const void* src, int rows, size_t row_bytes, int bpp, void* dst) {
    if (!src || !dst || rows < 0 || bpp < 1 || bpp > 8) {
        fn2::set_error("png_unfilter: null buffer, negative row count or bpp %d outside 1..8", bpp);
        return FN2_ERR_INVALID;
    }
    const uint8_t* in = static_cast<const uint8_t*>(src);
    uint8_t* out = static_cast<uint8_t*>(dst);
    const size_t n = row_bytes, k = (size_t)bpp;
    for (int y = 0; y < rows; y++) {
        const uint8_t* f = in + (size_t)y * (n + 1);
        const uint8_t* s = f + 1;
        uint8_t* d = out + (size_t)y * n;
        const uint8_t* up = y ? d - n : nullptr;                       // the row above, reconstructed; zeros for the first
        switch (f[0]) {
        case 0: memcpy(d, s, n); break;
        case 1:
            for (size_t i = 0; i < n; i++) d[i] = (uint8_t)(s[i] + (i >= k ? d[i - k] : 0));
            break;
        case 2:
            for (size_t i = 0; i < n; i++) d[i] = (uint8_t)(s[i] + (up ? up[i] : 0));
            break;
        case 3:
            for (size_t i = 0; i < n; i++) d[i] = (uint8_t)(s[i] + (((i >= k ? d[i - k] : 0) + (up ? up[i] : 0)) >> 1));
            break;
        case 4:
            for (size_t i = 0; i < n; i++) {
                const int a = i >= k ? d[i - k] : 0, b = up ? up[i] : 0, c = up && i >= k ? up[i - k] : 0;
                d[i] = (uint8_t)(s[i] + paeth(a, b, c));
            }
            break;
        default:
            fn2::set_error("png_unfilter: row %d has filter type %d (PNG defines 0 to 4)", y, (int)f[0]);
            return FN2_ERR_INVALID;
        }
    }
    return FN2_OK;
}
