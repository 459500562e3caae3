// TEST INFRASTRUCTURE — host emulation of csnet_salmetric_images_u8 (sod100k_b200/csrc/image_io.cuh).
//
// Computes each map byte with the device function the kernel calls (img_out_value) and counts it against the GT the way the
// kernel does, so `-m "not gpu"` tests can check the counting against oracle/salmetric.py without a GPU.
#define CSNET_HOST_EMU 1
#include <cstdint>
#include <cstring>

#include "../../sod100k_b200/csrc/image_io.cuh"

// fp32 logits [H][W] and a uint8 GT [h][w] -> hist_all[256], hist_pos[256], abs_sum and the uint8 map [h][w].
extern "C" void csnet_emu_salmetric_image(const float* z, int H, int W, const uint8_t* gt, int h, int w, uint32_t* hist_all,
                                          uint32_t* hist_pos, uint64_t* abs_sum, uint8_t* map) {
  std::memset(hist_all, 0, 256 * sizeof(uint32_t));
  std::memset(hist_pos, 0, 256 * sizeof(uint32_t));
  uint64_t d = 0;
  for (int oy = 0; oy < h; ++oy) {
    const csnet::ImgTap ty = csnet::img_tap(oy, H, h);
    for (int ox = 0; ox < w; ++ox) {
      const int64_t p = (int64_t)oy * w + ox;
      const uint8_t q = csnet::img_out_value(z, W, ty, csnet::img_tap(ox, W, w));
      const int t = gt[p];
      map[p] = q;
      ++hist_all[q];
      if (t > 128) ++hist_pos[q];
      d += (uint64_t)(q > t ? q - t : t - q);
    }
  }
  *abs_sum = d;
}
