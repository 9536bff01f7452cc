// The pixel formulas of the reference's video frames (radiance_fields/video_utils.py:28-34,334-366,471-627 and
// utils/visualization_tools.py:30-33,79-156), stated once for csrc/video.cu.  The build passes -fmad=false, and every
// operation below is written with its rounding, as numpy rounds it:
//   * to8b: (255 * np.clip(x, 0, 1)).astype(np.uint8) -- the product in the dtype the frame reached to8b in (float64
//     once np.concatenate met a depth row, whose colours are float64; float32 otherwise), then truncation; NaN
//     survives np.clip and its cast gives 0;
//   * the blend: a * alpha + b * (1 - alpha) on float32 arrays, then np.clip;
//   * the depth colour: numpy 2's promotion (the float32 curve minus a float64 bound is float64), matplotlib 3.6.1's
//     Colormap.__call__ index rule, and a turbo table already passed through to8b.
#pragma once
#include <stdint.h>

namespace emer {

// -np.log(4.0 + 1e-6) and -np.log(120 + 1e-6) in float64: the curved lo and hi of depth_visualizer
constexpr double VIDEO_DEPTH_CURVE_LO = -0x1.62e43421617e5p+0;
constexpr double VIDEO_DEPTH_CURVE_HI = -0x1.326643cd3a42cp+2;
constexpr double VIDEO_DEPTH_MIN = VIDEO_DEPTH_CURVE_HI;                           // np.minimum(lo, hi)
constexpr double VIDEO_DEPTH_SPAN = VIDEO_DEPTH_CURVE_LO - VIDEO_DEPTH_CURVE_HI;   // np.abs(hi - lo)

__device__ __forceinline__ uint8_t video_to8b_f32(float x) {
    if (!(x == x)) return 0;
    x = x < 0.0f ? 0.0f : (x > 1.0f ? 1.0f : x);
    return (uint8_t)__float2int_rz(__fmul_rn(255.0f, x));
}

__device__ __forceinline__ uint8_t video_to8b_f64(double x) {
    if (!(x == x)) return 0;
    x = x < 0.0 ? 0.0 : (x > 1.0 ? 1.0 : x);
    return (uint8_t)__double2int_rz(__dmul_rn(255.0, x));
}

// float32 product x to uint8, the product widened to float64 first when the frame is float64 (exact)
__device__ __forceinline__ uint8_t video_to8b(float x, bool f64) {
    return f64 ? video_to8b_f64((double)x) : video_to8b_f32(x);
}

// np.clip(a * alpha + b * (1 - alpha), 0, 1) on float32 arrays (NaN kept)
__device__ __forceinline__ float video_blend(float a, float alpha, float b) {
    const float v = __fadd_rn(__fmul_rn(a, alpha), __fmul_rn(b, __fsub_rn(1.0f, alpha)));
    return v < 0.0f ? 0.0f : (v > 1.0f ? 1.0f : v);
}

// The turbo entry of one depth pixel, or -1 for matplotlib's "bad" colour (black after to8b).  The curve
// -np.log(depth + 1e-6) is float32 (numpy's float32 log, here the float64 log rounded once); the normalisation, the
// clip, nan_to_num and the opacity product are float64; the index is min(int(v * 256), 255), 0 below 0.
__device__ __forceinline__ int video_depth_index(float depth, float opacity) {
    const float x = __fadd_rn(depth, 1e-6f);
    const float curve = -__double2float_rn(log((double)x));
    double v = __ddiv_rn(__dsub_rn((double)curve, VIDEO_DEPTH_MIN), VIDEO_DEPTH_SPAN);
    v = v < 0.0 ? 0.0 : (v > 1.0 ? 1.0 : v);             // np.clip keeps NaN ...
    if (!(v == v)) v = 0.0;                               // ... and np.nan_to_num zeroes it
    v = __dmul_rn(v, (double)opacity);                    // value *= weight
    if (!(v == v)) return -1;                             // a NaN or infinite opacity: "bad"
    const double s = __dmul_rn(v, 256.0);
    if (s < 0.0) return 0;                                // under: the first colour
    if (s >= 256.0) return 255;                           // v == 1 and over: the last colour
    return __double2int_rz(s);
}

}  // namespace emer
