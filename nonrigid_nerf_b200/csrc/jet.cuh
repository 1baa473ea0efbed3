// matplotlib's cm.jet as the colour images use it: LinearSegmentedColormap("jet", _jet_data, N=256), as float64, fp32 and
// to8b tables built at compile time, and one __constant__ copy of the fp32 and uint8 tables per translation unit that
// includes this header (eval.cu, lpips.cu).
//
// _jet_data as matplotlib publishes it (matplotlib/_cm.py): per channel the breakpoints x with the values y0 (left of x)
// and y1 (right of x).  The table is what matplotlib's _create_lookup_table makes of it, in the same float64 operations:
// xind = 255 * (i * (1 / 255)), k = searchsorted(255 * x, xind), lut = (xind - 255 x[k-1]) / (255 x[k] - 255 x[k-1])
// * (y0[k] - y1[k-1]) + y1[k-1], the ends y1[0] and y0[-1], clipped to [0, 1].
#pragma once
#include <stdint.h>

namespace nrn {
namespace {

struct JetSegments {
  int n;
  double x[6], y0[6], y1[6];
};
constexpr JetSegments kJetRed{5, {0.0, 0.35, 0.66, 0.89, 1.0}, {0, 0, 1, 1, 0.5}, {0, 0, 1, 1, 0.5}};
constexpr JetSegments kJetGreen{6, {0.0, 0.125, 0.375, 0.64, 0.91, 1.0}, {0, 0, 1, 1, 0, 0}, {0, 0, 1, 1, 0, 0}};
constexpr JetSegments kJetBlue{5, {0.0, 0.11, 0.34, 0.65, 1.0}, {0.5, 1, 1, 0, 0}, {0.5, 1, 1, 0, 0}};

constexpr double clip01(double v) { return v < 0.0 ? 0.0 : (v > 1.0 ? 1.0 : v); }

constexpr double jet_entry(const JetSegments& s, int i) {
  if (i == 0) return clip01(s.y1[0]);
  if (i == 255) return clip01(s.y0[s.n - 1]);
  const double xind = 255.0 * (i * (1.0 / 255.0));
  int k = 0;
  while (s.x[k] * 255.0 < xind) ++k;   // searchsorted, side="left"
  const double x0 = s.x[k - 1] * 255.0, x1 = s.x[k] * 255.0;
  const double distance = (xind - x0) / (x1 - x0);
  return clip01(distance * (s.y0[k] - s.y1[k - 1]) + s.y1[k - 1]);
}

struct JetTables {
  double rgb[256 * 3];    // cm.jet(i)[:3]
  float rgbf[256 * 3];    // the same in fp32: the colour images
  uint8_t rgb8[256 * 3];  // to8b(cm.jet(i)[:3]) = uint8(255 * clip(c, 0, 1)): the error images
};
constexpr JetTables make_jet_tables() {
  JetTables t{};
  const JetSegments* seg[3] = {&kJetRed, &kJetGreen, &kJetBlue};
  for (int i = 0; i < 256; ++i)
    for (int c = 0; c < 3; ++c) {
      const double v = jet_entry(*seg[c], i);
      t.rgb[i * 3 + c] = v;
      t.rgbf[i * 3 + c] = static_cast<float>(v);
      t.rgb8[i * 3 + c] = static_cast<uint8_t>(255.0 * clip01(v));
    }
  return t;
}
constexpr JetTables kJet = make_jet_tables();

struct JetDeviceTables {
  float rgbf[256 * 3];
  uint8_t rgb8[256 * 3];
};
constexpr JetDeviceTables make_jet_device_tables() {
  JetDeviceTables t{};
  for (int i = 0; i < 256 * 3; ++i) { t.rgbf[i] = kJet.rgbf[i]; t.rgb8[i] = kJet.rgb8[i]; }
  return t;
}
__constant__ JetDeviceTables c_jet = make_jet_device_tables();

}  // namespace
}  // namespace nrn
