// TEST HARNESS ONLY (never loaded by the product): the half-precision clip-storage scan of gather_kernels.cu
// (pp_img_prop_scan_u8h) on the host.  The per-pixel rules are pp_elem.cuh's, compiled for the host; the loops here play
// the role of the CUDA grid and mirror the launcher step for step, and hs_rn16 plays __float2half_rn.
#define PP_HOSTSIM 1
#include <cstring>
#include <vector>
#include "../../propainter_b200/csrc/pp_elem.cuh"

// float -> IEEE binary16, round to nearest even (overflow to inf, NaN kept quiet)
static uint16_t hs_rn16(float f) {
  uint32_t x;
  memcpy(&x, &f, 4);
  const uint16_t sign = (uint16_t)((x >> 16) & 0x8000u);
  const uint32_t ax = x & 0x7fffffffu;
  if (ax > 0x7f800000u) return sign | 0x7e00u;
  if (ax >= 0x477ff000u) return sign | 0x7c00u;               // >= 65520 rounds to inf
  if (ax < 0x38800000u) {                                      // below 2^-14: a multiple of 2^-24, scaled exactly
    float a;
    memcpy(&a, &ax, 4);
    return sign | (uint16_t)nearbyintf(a * 16777216.0f);
  }
  uint32_t h = (((ax >> 23) - 112u) << 10) | ((ax & 0x7fffffu) >> 13);
  const uint32_t rem = ax & 0x1fffu;
  if (rem > 0x1000u || (rem == 0x1000u && (h & 1u))) ++h;      // a carry into the exponent is the right result
  return sign | (uint16_t)h;
}

// k_imgprop_step_u8h over all pixels
static void hs_step(int H, int W, const uint8_t* u8, const float* md, const float* cur, const float* mcur, const float* prev,
                    const float* mprev, const pp_half* fprop, const pp_half* fcheck, float* out, float* mout, uint16_t* out16,
                    uint16_t* mout16, int nearest) {
  const int HW = H * W;
  for (int pix = 0; pix < HW; ++pix) {
    const float m = md[pix];
    float fr[3], cv[3], ov[3];
    for (int c = 0; c < 3; ++c) {
      fr[c] = pp_u8_frame(u8[3 * (long)pix + c]);
      cv[c] = cur ? cur[(long)c * HW + pix] : PP_MUL(fr[c], PP_SUB(1.0f, m));
    }
    float mo = mcur ? mcur[pix] : m;
    if (prev) mo = pp_imgprop_values(pix, H, W, cv, mo, prev, mprev, fprop, fcheck, ov, nearest);
    else for (int c = 0; c < 3; ++c) ov[c] = cv[c];
    if (out) {
      for (int c = 0; c < 3; ++c) out[(long)c * HW + pix] = ov[c];
      mout[pix] = mo;
    }
    if (out16) {
      for (int c = 0; c < 3; ++c) out16[(long)c * HW + pix] = hs_rn16(pp_imgprop_compose(fr[c], ov[c], m));
      mout16[pix] = hs_rn16(mo);
    }
  }
}

extern "C" {

uint16_t hs_float_to_half(float f) { return hs_rn16(f); }
float hs_half_to_float(uint16_t h) { pp_half v = {h}; return pp_widen(v); }

// pp_img_prop_scan_u8h: frames_u8 [t][H][W][3], masks [t][H][W], flows fp16 bits [t-1][2][H][W] -> fp16 bits of frames
// [lo, hi): of [hi-lo][3][H][W], om [hi-lo][H][W]
void hs_img_prop_scan_u8h(const uint8_t* u8, const float* masks, const uint16_t* flows_f, const uint16_t* flows_b, uint16_t* of,
                          uint16_t* om, int t, int H, int W, int lo, int hi, int nearest) {
  if (lo >= hi) return;
  const long HW = (long)H * W;
  const pp_half* ff = reinterpret_cast<const pp_half*>(flows_f);
  const pp_half* fb = reinterpret_cast<const pp_half*>(flows_b);
  std::vector<float> bf((size_t)t * 3 * HW), bm((size_t)t * HW), rf(2 * 3 * HW), rm(2 * HW);
  hs_step(H, W, u8 + (t - 1) * 3 * HW, masks + (t - 1) * HW, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
          &bf[(size_t)(t - 1) * 3 * HW], &bm[(size_t)(t - 1) * HW], nullptr, nullptr, nearest);
  for (int i = t - 2; i >= 0; --i)
    hs_step(H, W, u8 + i * 3 * HW, masks + i * HW, nullptr, nullptr, &bf[(size_t)(i + 1) * 3 * HW], &bm[(size_t)(i + 1) * HW],
            ff + i * 2 * HW, fb + i * 2 * HW, &bf[(size_t)i * 3 * HW], &bm[(size_t)i * HW], nullptr, nullptr, nearest);
  if (lo == 0)
    hs_step(H, W, u8, masks, bf.data(), bm.data(), nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, of, om, nearest);
  for (int i = 1; i < hi; ++i) {
    const float* pf = i == 1 ? bf.data() : &rf[(size_t)((i - 1) & 1) * 3 * HW];
    const float* pm = i == 1 ? bm.data() : &rm[(size_t)((i - 1) & 1) * HW];
    const bool keep = i >= lo;
    hs_step(H, W, u8 + i * 3 * HW, masks + i * HW, &bf[(size_t)i * 3 * HW], &bm[(size_t)i * HW], pf, pm, fb + (i - 1) * 2 * HW,
            ff + (i - 1) * 2 * HW, &rf[(size_t)(i & 1) * 3 * HW], &rm[(size_t)(i & 1) * HW],
            keep ? of + (i - lo) * 3 * HW : nullptr, keep ? om + (i - lo) * HW : nullptr, nearest);
  }
}
}
