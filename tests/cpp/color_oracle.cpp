// color_oracle.cpp — sequential CPU restatement of the camera-coloured and IMU-frame publishers, to the contract of
// DESIGN.md §9 (test infrastructure; loaded by tests/color_oracle.py, built with g++ -ffp-contract=off):
//   publish_frame_world_color   src/laserMapping.cpp:323-381 (paramSetting :279-289 for the matrices)
//   RGBpointBodyLidarToIMU      src/laserMapping.cpp:1113-1122 (publish_frame_body :1543-1558)
// Written as the reference's loops are, point by point, with the undefined int conversion replaced by the contract's
// rejection of non-finite or non-int32 pixel coordinates.
#include <cmath>
#include <cstdint>

namespace {

struct V3 { double x, y, z; };

// Eigen's q * v (_transformVector): uv = 2 (q.vec × v); v + w·uv + q.vec × uv
V3 qrot(const double* q, V3 v) {
  V3 uv{q[1] * v.z - q[2] * v.y, q[2] * v.x - q[0] * v.z, q[0] * v.y - q[1] * v.x};
  uv.x = uv.x + uv.x; uv.y = uv.y + uv.y; uv.z = uv.z + uv.z;
  const V3 c{q[1] * uv.z - q[2] * uv.y, q[2] * uv.x - q[0] * uv.z, q[0] * uv.y - q[1] * uv.x};
  return V3{(v.x + q[3] * uv.x) + c.x, (v.y + q[3] * uv.y) + c.y, (v.z + q[3] * uv.z) + c.z};
}

// state26: pos 0-2, rot 3-6 (x,y,z,w), offset_R_L_I 7-10, offset_T_L_I 11-13
V3 lidar_to_imu(const double* st, float x, float y, float z) {
  V3 a = qrot(st + 7, V3{x, y, z});
  return V3{a.x + st[11], a.y + st[12], a.z + st[13]};
}

// trunc toward zero when the value is finite and representable in int32
bool to_int(double d, int* out) {
  if (!std::isfinite(d) || !(d > -2147483649.0) || !(d < 2147483648.0)) return false;
  *out = (int)d;
  return true;
}

}  // namespace

extern "C" {

// M = cam_in (3x4) · cam_ex (4x4), each element summed over k = 0..3 in index order
void orc_projection(const double* cam_ex, const double* cam_in, double* M) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) {
      double s = 0.0;
      for (int k = 0; k < 4; ++k) s = k == 0 ? cam_in[4 * r] * cam_ex[c] : s + cam_in[4 * r + k] * cam_ex[4 * k + c];
      M[4 * r + c] = s;
    }
}

// pts: n × (x, y, z, intensity) float, lidar frame; img: H × W × 3 bgr8, row pitch 3·W.  Writes the kept points' world
// x, y, z, intensity, their colour word (b | g << 8 | r << 16 | 255 << 24) and source index; returns the kept count.
int orc_colorize(const double* cam_ex, const double* cam_in, int W, int H, const unsigned char* img, const float* pts, int n,
                 const double* st, float* out_xyzi, unsigned* out_bgra, int* out_idx) {
  double M[12];
  orc_projection(cam_ex, cam_in, M);
  int k = 0;
  for (int i = 0; i < n; ++i) {
    const float* p = pts + 4 * (size_t)i;
    const double cloud[4] = {p[0], p[1], p[2], 1};
    double cam[3];
    for (int r = 0; r < 3; ++r) {
      double s = M[4 * r] * cloud[0];
      for (int c = 1; c < 4; ++c) s = s + M[4 * r + c] * cloud[c];
      cam[r] = s;
    }
    int px, py;
    if (!to_int(cam[0] / cam[2], &px) || !to_int(cam[1] / cam[2], &py)) continue;
    if (!(px >= 0 && px < W && py >= 0 && py < H && p[0] > 0)) continue;
    const unsigned char* b = img + 3 * ((size_t)py * W + px);
    // world: rot · (offR · p + offT) + pos, rounded to float
    const V3 a = lidar_to_imu(st, p[0], p[1], p[2]);
    const V3 g = qrot(st + 3, a);
    out_xyzi[4 * (size_t)k + 0] = (float)(g.x + st[0]);
    out_xyzi[4 * (size_t)k + 1] = (float)(g.y + st[1]);
    out_xyzi[4 * (size_t)k + 2] = (float)(g.z + st[2]);
    out_xyzi[4 * (size_t)k + 3] = p[3];
    out_bgra[k] = (unsigned)b[0] | ((unsigned)b[1] << 8) | ((unsigned)b[2] << 16) | (255u << 24);
    out_idx[k] = i;
    ++k;
  }
  return k;
}

// imageCallback's loop (:254-260): the top-left H × W window of a bgr8 image with row step `step`, pixel by pixel
void orc_copy_image(const unsigned char* src, int step, int W, int H, unsigned char* dst) {
  for (int row = 0; row < H; ++row)
    for (int col = 0; col < W; ++col)
      for (int c = 0; c < 3; ++c) dst[3 * ((size_t)row * W + col) + c] = src[(size_t)row * step + 3 * col + c];
}

void orc_to_imu(const float* pts, int n, const double* st, float* out) {
  for (int i = 0; i < n; ++i) {
    const float* p = pts + 4 * (size_t)i;
    const V3 a = lidar_to_imu(st, p[0], p[1], p[2]);
    out[4 * (size_t)i + 0] = (float)a.x;
    out[4 * (size_t)i + 1] = (float)a.y;
    out[4 * (size_t)i + 2] = (float)a.z;
    out[4 * (size_t)i + 3] = p[3];
  }
}

}  // extern "C"
