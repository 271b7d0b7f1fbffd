// The 11-tap Gaussian of the SSIM window (utils/util.py:217: cv2.getGaussianKernel(11, 1.5), the window is its outer
// product), shared by the uint8 evaluation metric (metrics.cu) and the fp32 training loss (ssim_loss.cu).
#pragma once

namespace binb {

// cv2.getGaussianKernel(11, 1.5) bit for bit (OpenCV's bit-exact kernel differs from exp()/sum in the last bits).
// Symmetric: kGauss11[t] == kGauss11[10 - t].  static: each translation unit holds its own copy.
static __constant__ double kGauss11[11] = {0x1.0d956b52a1d6ep-10, 0x1.f1fe01ae5a5b5p-8, 0x1.26eb175d83f66p-5,
                                           0x1.bff0fe8e98418p-4,  0x1.b43c3f52b19f3p-3, 0x1.106560aa892bfp-2,
                                           0x1.b43c3f52b19f3p-3,  0x1.bff0fe8e98418p-4, 0x1.26eb175d83f66p-5,
                                           0x1.f1fe01ae5a5b5p-8,  0x1.0d956b52a1d6ep-10};

}  // namespace binb
