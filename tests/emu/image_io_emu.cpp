// TEST INFRASTRUCTURE — host emulation of the image resize kernels (sod100k_b200/csrc/image_io.cuh).
//
// Compiles the same per-pixel functions the two kernels run and walks one image the way they do, so `-m "not gpu"` tests can
// check the resize arithmetic against scipy.ndimage.zoom without a GPU.
#define CSNET_HOST_EMU 1
#include <cstdint>

#include "../../sod100k_b200/csrc/image_io.cuh"

// uint8 [h][w][3] -> fp32 [3][H][W], normalised with mean / std (float[3], as the C ABI takes them).
extern "C" void csnet_emu_resize_in(const uint8_t* img, int h, int w, int H, int W, const float* mean, const float* stdv, float* out) {
  double tab[256];
  for (int i = 0; i < 256; ++i) tab[i] = (double)i / 255.0;
  for (int oy = 0; oy < H; ++oy) {
    const csnet::ImgTap ty = csnet::img_tap(oy, h, H);
    for (int ox = 0; ox < W; ++ox) {
      const csnet::ImgTap tx = csnet::img_tap(ox, w, W);
      for (int c = 0; c < 3; ++c)
        out[((int64_t)c * H + oy) * W + ox] = csnet::img_in_value(img, w, tab, ty, tx, c, (double)mean[c], (double)stdv[c]);
    }
  }
}

// fp32 logits [H][W] -> uint8 map [h][w].
extern "C" void csnet_emu_resize_out(const float* z, int H, int W, int h, int w, uint8_t* out) {
  for (int oy = 0; oy < h; ++oy) {
    const csnet::ImgTap ty = csnet::img_tap(oy, H, h);
    for (int ox = 0; ox < w; ++ox) out[(int64_t)oy * w + ox] = csnet::img_out_value(z, W, ty, csnet::img_tap(ox, W, w));
  }
}

extern "C" void csnet_emu_sigmoid(const float* z, int64_t n, float* s) {
  for (int64_t i = 0; i < n; ++i) s[i] = csnet::img_sigmoid(z[i]);
}
