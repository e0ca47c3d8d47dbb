// scan_step_emul.cpp — TEST-ONLY: the ballot resolution of the warp post-filter scans (pf_scan_step_d, ext_device.cuh) compiled for the
// host, applied step by step as pf_scan_warp (pipeline.cu) applies it.  Never part of the product.
#include "ext_device.cuh"

extern "C" {

// The warp scan of box kinds kind[0..n) (0 skipped, 1 counted, 2 hit) with lim: the masks of each 32-box step resolved by pf_scan_step_d
// in order.  Returns v; *stop_step = the step the scan stopped in, -1 when it ran off the end or never started.
int scan_step_emul(const int8_t *kind, int n, int lim, int *stop_step) {
    int v = 0;
    *stop_step = -1;
    for (int i0 = 0; i0 < n && v < lim; i0 += 32) {
        uint32_t cm = 0, hm = 0;
        for (int j = 0; j < 32 && i0 + j < n; ++j) { cm |= (uint32_t) (kind[i0 + j] == 1) << j; hm |= (uint32_t) (kind[i0 + j] == 2) << j; }
        if (pf_scan_step_d(cm, hm, v, lim)) { *stop_step = i0 / 32; break; }
    }
    return v;
}

}
