// TEST INFRASTRUCTURE — host build of CSF+Res2Net's per-pixel training-sample functions (sod100k_b200/csrc/image_io.cuh).
//
// csf_train_batch_u8_kernel calls exactly these functions, so `-m "not gpu"` tests can check them against the reference's
// ImageDataTrain golden without a GPU.
#define CSNET_HOST_EMU 1
#include <cstdint>

#include "../../sod100k_b200/csrc/image_io.cuh"

// One training sample as csf_train_batch_u8_kernel builds it: image uint8 [h][w][3], mask uint8 [h][w] -> x fp32 [3][h][w] and
// t fp32 [h][w], both flipped along W when flip is 1 (img_csf_src_col, img_csf_in_value, img_csf_label_value).
extern "C" void csnet_emu_csf_train_sample(const uint8_t* img, const uint8_t* mask, int h, int w, int flip, const double* mean,
                                           const double* stdv, float* x, float* t) {
  const int64_t hw = (int64_t)h * w;
  for (int oy = 0; oy < h; ++oy)
    for (int ox = 0; ox < w; ++ox) {
      const int64_t p = (int64_t)oy * w + ox, q = (int64_t)oy * w + csnet::img_csf_src_col(ox, w, flip);
      for (int c = 0; c < 3; ++c) x[c * hw + p] = csnet::img_csf_in_value(img[3 * q + c], mean[c], stdv[c]);
      t[p] = csnet::img_csf_label_value(mask[q]);
    }
}
