// TEST INFRASTRUCTURE — host emulation of the training-data kernels (train_batch_u8_kernel, val_mae_u8_kernel in
// sod100k_b200/csrc/image_io.cuh).
//
// Compiles the same per-pixel functions the kernels run and walks one sample the way they do.  Built with FMA contraction
// (tests/emu/train_data.py), as nvcc builds the kernels, so the training batch has the device's bits.
#define CSNET_HOST_EMU 1
#include <cstdint>

#include "../../sod100k_b200/csrc/image_io.cuh"

// One training sample: the stored uint8 image [h][w][3] and mask [h][w], the crop window (y0, x0, ch, cw) and the flip (0 none,
// 1 'lr', 2 'ud') -> fp32 input [3][H][W] and target [H][W].
extern "C" void csnet_emu_train_sample(const uint8_t* img, const uint8_t* mask, int w, int y0, int x0, int ch, int cw, int flip, int H,
                                       int W, const float* mean, const float* stdv, float* x, float* target) {
  double tab[256];
  for (int i = 0; i < 256; ++i) tab[i] = (double)i / 255.0;
  for (int oy = 0; oy < H; ++oy) {
    const csnet::ImgTap ty = csnet::img_tap_crop(csnet::img_tap(oy, ch, H), y0, ch, flip == 2);
    for (int ox = 0; ox < W; ++ox) {
      const csnet::ImgTap tx = csnet::img_tap_crop(csnet::img_tap(ox, cw, W), x0, cw, flip == 1);
      for (int c = 0; c < 3; ++c)
        x[((int64_t)c * H + oy) * W + ox] = csnet::img_in_value(img, w, tab, ty, tx, c, (double)mean[c], (double)stdv[c]);
      target[(int64_t)oy * W + ox] = csnet::img_mask_value(mask, w, tab, ty, tx);
    }
  }
}

// Validation MAE of one image: fp32 logits [H][W], uint8 GT [h][w]; the pixel terms summed in double in raster order.
extern "C" double csnet_emu_val_mae(const float* z, int H, int W, const uint8_t* gt, int h, int w) {
  const float sy = (float)H / (float)h, sx = (float)W / (float)w;
  double sum = 0.0;
  for (int oy = 0; oy < h; ++oy) {
    const csnet::MaeTap ty = csnet::mae_tap(oy, H, sy);
    for (int ox = 0; ox < w; ++ox) sum += (double)csnet::img_mae_term(z, W, ty, csnet::mae_tap(ox, W, sx), gt[(int64_t)oy * w + ox]);
  }
  return sum / ((double)h * (double)w);
}
