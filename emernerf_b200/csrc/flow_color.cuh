// The colour of one scene flow: the reference's scene_flow_to_rgb (utils/visualization_tools.py:204-275) restated op
// for op as torch's CUDA kernels run it, one rounding per torch op (this library is compiled with -fmad=false, and
// every rounding is spelled with an intrinsic anyway).  Only the flow's x and y enter the colour.
//
//   complex flow   x + 1j*y: the complex product (y + 0i)(0 + 1i), then x added to its real part.  Its real part is
//                  y*0 - 0*1, so an infinite y gives NaN.  (torch's add also multiplies by alpha = 1 + 0i, which only
//                  changes signs of zero at radius 0, where the colour does not depend on the angle.)
//   radius, angle  hypotf and atan2f (thrust's abs and arg); angle += 2pi where angle < 0; angle *= 54 / (2pi)
//   scaling        FLOW_SCALE_HOST: radius * (1 / r) for a host radius r > 0 (torch's CUDA division by a host scalar
//                  multiplies by the fp32 reciprocal); FLOW_SCALE_DEVICE: radius / r for a device radius, when r > 0
//   hue            fmod(angle, 1), trunc, ceil, and a lerp of the 56-entry wheel (55 hues, then the first again)
//   background     bright: 255 - radius (255 - hue), and hue * (1 / radius) where radius > 1; dark: hue * radius, and
//                  255 - (1 / radius)(255 - hue) where radius > 1; then * (1 / 255.0f)
//
// A NaN radius or angle would index the wheel out of range in the reference (a device-side assert); here it gives NaN
// in all three channels.  An infinite radius follows the formula (1 / inf = 0).
#pragma once
#include "common.cuh"

namespace emer {

enum FlowScale { FLOW_SCALE_NONE = 0, FLOW_SCALE_HOST = 1, FLOW_SCALE_DEVICE = 2 };

constexpr int FLOW_WHEEL_COLS = 55;          // the reference's N_COLS: transitions 15, 6, 4, 11, 13, 6

struct FlowWheel {
    float c[FLOW_WHEEL_COLS + 1][3];
};

// The reference's _make_colorwheel: per transition, np.linspace(hue_from, hue_to, length, endpoint=False) stored as
// uint8.  Every transition moves one channel, so numpy takes its zero-step branch, ((double)i / length) * delta + from,
// and the uint8 store truncates.  Row 55 repeats row 0 (the cyclic wheel).
constexpr FlowWheel make_flow_wheel() {
    const int lengths[6] = {15, 6, 4, 11, 13, 6};
    const int hues[7][3] = {{255, 0, 0}, {255, 255, 0}, {0, 255, 0}, {0, 255, 255}, {0, 0, 255}, {255, 0, 255},
                            {255, 0, 0}};
    FlowWheel w{};
    int row = 0;
    for (int t = 0; t < 6; ++t)
        for (int i = 0; i < lengths[t]; ++i, ++row)
            for (int a = 0; a < 3; ++a) {
                const double delta = (double)(hues[t + 1][a] - hues[t][a]);
                w.c[row][a] = (float)(int)((double)i / (double)lengths[t] * delta + (double)hues[t][a]);
            }
    for (int a = 0; a < 3; ++a) w.c[FLOW_WHEEL_COLS][a] = w.c[0][a];
    return w;
}

static __constant__ FlowWheel kFlowWheel = make_flow_wheel();

// The radius and angle of the complex flow x + 1j*y, as torch.abs and torch.angle give them.
__device__ __forceinline__ void flow_polar(float x, float y, float& radius, float& angle) {
    const float re = __fadd_rn(x, __fsub_rn(__fmul_rn(y, 0.0f), __fmul_rn(0.0f, 1.0f)));
    const float im = __fadd_rn(0.0f, __fadd_rn(__fmul_rn(y, 1.0f), __fmul_rn(0.0f, 0.0f)));
    radius = hypotf(re, im);
    angle = atan2f(im, re);
}

// rgb = scene_flow_to_rgb of the flow (x, y, .).  scale: the fp32 reciprocal of the host radius (FLOW_SCALE_HOST) or
// the device radius (FLOW_SCALE_DEVICE); ignored for FLOW_SCALE_NONE.
__device__ __forceinline__ void flow_rgb(float x, float y, int scale_mode, float scale, bool bright, float rgb[3]) {
    float radius, angle;
    flow_polar(x, y, radius, angle);
    if (scale_mode == FLOW_SCALE_HOST) radius = __fmul_rn(radius, scale);
    else if (scale_mode == FLOW_SCALE_DEVICE && scale > 0.0f) radius = __fdiv_rn(radius, scale);
    if (angle < 0.0f) angle = __fadd_rn(angle, 6.2831855f);                     // (float)(2 * np.pi)
    angle = __fmul_rn(angle, (float)(54.0 / 6.283185307179586));               // (N_COLS - 1) / (2 * np.pi)
    if (radius != radius || angle != angle) {
        rgb[0] = rgb[1] = rgb[2] = __int_as_float(0x7fffffff);
        return;
    }
    const float frac = fmodf(angle, 1.0f);
    const int i0 = min(max((int)truncf(angle), 0), FLOW_WHEEL_COLS);
    const int i1 = min(max((int)ceilf(angle), 0), FLOW_WHEEL_COLS);
    const float keep = __fsub_rn(1.0f, frac);
    const bool over = radius > 1.0f;
    const float inv = over ? __fdiv_rn(1.0f, radius) : 0.0f;                  // torch: reciprocal(radius) * 1
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float hue = __fadd_rn(__fmul_rn(kFlowWheel.c[i0][a], keep), __fmul_rn(kFlowWheel.c[i1][a], frac));
        float c;
        if (bright) c = over ? __fmul_rn(hue, inv) : __fsub_rn(255.0f, __fmul_rn(radius, __fsub_rn(255.0f, hue)));
        else c = over ? __fsub_rn(255.0f, __fmul_rn(inv, __fsub_rn(255.0f, hue))) : __fmul_rn(hue, radius);
        rgb[a] = __fmul_rn(c, 1.0f / 255.0f);                                  // / 255.0: times the fp32 reciprocal
    }
}

}  // namespace emer
