// TEST INFRASTRUCTURE — host build of CSF+Res2Net's per-pixel test-path functions (sod100k_b200/csrc/image_io.cuh).
//
// csf_input_u8_kernel and the CsfMap instances of the map and SalMetric kernels call exactly these functions, so `-m "not gpu"`
// tests can check them against the reference's numpy / cv2 goldens without a GPU.
#define CSNET_HOST_EMU 1
#include <cstdint>

#include "../../sod100k_b200/csrc/image_io.cuh"

// uint8 [h][w][3] -> fp32 [3][h][w] (img_csf_in_value), mean / std double[3].
extern "C" void csnet_emu_csf_input(const uint8_t* img, int h, int w, const double* mean, const double* stdv, float* out) {
  const int64_t hw = (int64_t)h * w;
  for (int64_t p = 0; p < hw; ++p)
    for (int c = 0; c < 3; ++c) out[c * hw + p] = csnet::img_csf_in_value(img[3 * p + c], mean[c], stdv[c]);
}

// Sigmoid values s[n] -> map bytes (img_csf_out_byte).
extern "C" void csnet_emu_csf_out_byte(const float* s, int64_t n, uint8_t* q) {
  for (int64_t i = 0; i < n; ++i) q[i] = csnet::img_csf_out_byte(s[i]);
}
