// CPU oracle of flb_keyframes_scan_context / flb_keyframes_scan_contexts: a literal sequential restatement of
// SCManager::makeScancontext (include/sc-relo/Scancontext.cpp:195-251) and xy2theta (:23-36) with the reference's types
// (PointType pt, float azim_angle / azim_range, double desc).  atan is the double ::atan, called on the float quotient.
// Test infrastructure only; compiled by tests/scan_context_oracle.py with
//   g++ -O2 -std=c++17 -fPIC -shared -ffp-contract=off -fno-fast-math
// (no FMA contraction, like the reference build and the -fmad=false device code).
//
// Besides the descriptor it reports which points are atan-sensitive: their float angle lies within 2 float ulps of a
// value in another sector, so an atan that differs from glibc's by an ulp or two (the device's) may bin them one sector
// over.  bin_mask marks every bin such a point could reach (its own sector and those of the angles within 2 ulps).
#include <algorithm>
#include <cmath>

namespace {

const int PC_NUM_RING = 20, PC_NUM_SECTOR = 60;
const double PC_MAX_RADIUS = 80.0;

struct PointType { float x, y, z; };

float xy2theta(const float& _x, const float& _y) {
  if ((_x >= 0) & (_y >= 0)) return (180 / M_PI) * ::atan((double)(_y / _x));
  else if ((_x < 0) & (_y >= 0)) return 180 - ((180 / M_PI) * ::atan((double)(_y / (-_x))));
  else if ((_x < 0) & (_y < 0)) return 180 + ((180 / M_PI) * ::atan((double)(_y / _x)));
  else return 360 - ((180 / M_PI) * ::atan((double)((-_y) / _x)));
}

int sector_of(float azim_angle) {
  // int(NaN) is INT_MIN on x86 (cvttsd2si); the clamp takes it to 1
  return std::max(std::min(PC_NUM_SECTOR, int(ceil((azim_angle / 360.0) * PC_NUM_SECTOR))), 1);
}

}  // namespace

extern "C" int orc_scan_context(const float* pts, int n, int stride_floats, double lidar_height, double* desc,
                                unsigned char* sensitive, unsigned char* bin_mask) {
  if (n < 0 || stride_floats < 3 || !desc) return 1;
  const int NO_POINT = -1000;
  for (int b = 0; b < PC_NUM_RING * PC_NUM_SECTOR; ++b) {
    desc[b] = NO_POINT;
    if (bin_mask) bin_mask[b] = 0;
  }
  PointType pt;
  float azim_angle, azim_range;
  int ring_idx, sctor_idx;
  for (int i = 0; i < n; ++i) {
    const float* p = pts + (size_t)i * stride_floats;
    if (sensitive) sensitive[i] = 0;
    pt.x = p[0];
    pt.y = p[1];
    pt.z = p[2] + lidar_height;
    azim_range = sqrt(pt.x * pt.x + pt.y * pt.y);
    azim_angle = xy2theta(pt.x, pt.y);
    if (azim_range > PC_MAX_RADIUS) continue;
    ring_idx = std::max(std::min(PC_NUM_RING, int(ceil((azim_range / PC_MAX_RADIUS) * PC_NUM_RING))), 1);
    sctor_idx = sector_of(azim_angle);
    double& bin = desc[(ring_idx - 1) * PC_NUM_SECTOR + (sctor_idx - 1)];
    if (bin < pt.z) bin = pt.z;
    if (!(pt.z > NO_POINT)) continue;   // touches nothing, whatever its sector
    bool sens = false;
    for (int dir = -1; dir <= 1; dir += 2) {
      float a = azim_angle;
      for (int step = 0; step < 2; ++step) {
        a = std::nextafter(a, dir * INFINITY);
        const int s = sector_of(a);
        if (s != sctor_idx) {
          sens = true;
          if (bin_mask) bin_mask[(ring_idx - 1) * PC_NUM_SECTOR + (s - 1)] = 1;
        }
      }
    }
    if (sens) {
      if (sensitive) sensitive[i] = 1;
      if (bin_mask) bin_mask[(ring_idx - 1) * PC_NUM_SECTOR + (sctor_idx - 1)] = 1;
    }
  }
  for (int b = 0; b < PC_NUM_RING * PC_NUM_SECTOR; ++b)
    if (desc[b] == NO_POINT) desc[b] = 0;
  return 0;
}
