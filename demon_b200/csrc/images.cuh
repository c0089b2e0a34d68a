// Image resizing on the device (images.cu): Pillow's `Image.resize` for RGB uint8, bit for bit, and adjust_intrinsics.
#pragma once
#include "common.cuh"

namespace demon {

// DEMON_E_INVALID (with a message naming `who`) unless 1 <= h, w, oh, ow <= 8192 and resample is NEAREST, BILINEAR or BICUBIC
int resize_u8_check(int h, int w, int oh, int ow, int resample, const char* who);

// Resizes n RGB uint8 images [h,w,3] (pixel stride 3, channel stride 1, `sy` bytes between rows) into dst [n,oh,ow,3]
// (contiguous).  Image z starts at src + (z / per) * s_outer + (z % per) * s_inner: per = 1 is a plain batch with sample
// stride s_outer, per = 2 the [B,2,h,w,3] image pairs of the pipeline.  The arguments must have passed resize_u8_check.
int resize_u8_launch(const uint8_t* src, int64_t s_outer, int64_t s_inner, int per, int64_t sy, int n, int h, int w, uint8_t* dst,
                     int oh, int ow, int resample, cudaStream_t stream);

// DEMON_E_INVALID unless 1 <= h, w, oh, ow <= 8192, h <= 100 w and knew = (fx, fy, cx, cy) has finite positive focal lengths
// and a finite principal point
int adjust_intrinsics_check(int h, int w, const double* knew, int oh, int ow, const char* who);

// adjust_intrinsics of n images addressed like resize_u8_launch's: image z, with intrinsics K[z] = (fx, fy, cx, cy) (device
// doubles, pixels), resized with BILINEAR or LANCZOS and cropped to the target intrinsics knew (host) and size ow x oh, into
// dst [n,oh,ow,3]; status[z] (device) = 0 ok, 1 fill added, 2 invalid K (all fill).  Arguments must have passed the check.
int adjust_intrinsics_launch(const uint8_t* src, int64_t s_outer, int64_t s_inner, int per, int64_t sy, int n, int h, int w, const double* K,
                             const double* knew, uint8_t* dst, int oh, int ow, uint8_t* status, cudaStream_t stream);

}  // namespace demon
