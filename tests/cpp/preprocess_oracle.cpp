// CPU oracle of flb_frontend_preprocess: a literal sequential restatement of Preprocess::process with feature extraction
// off (src/preprocess.cpp livox_handler :178-204, velodyne_handler :302-340 + :417-473, oust64_handler :271-297), over
// the same driver-record layouts the C ABI takes.  Test infrastructure only; compiled by tests/preprocess_oracle.py with
//   g++ -O2 -std=c++17 -fPIC -shared -ffp-contract=off -fno-fast-math -Iinclude
// (no FMA contraction, like the reference build and the -fmad=false device code).
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "fastlio_b200.h"

namespace {

struct Pt { float x, y, z, intensity, curvature; };

template <class T>
T field(const unsigned char* rec, int off) {   // pcl::fromROSMsg: a field with no match reads as 0
  T v = T(0);
  if (off >= 0) std::memcpy(&v, rec + off, sizeof(T));
  return v;
}

float time_unit_scale(int unit) {   // Preprocess::process (:65-82)
  switch (unit) {
    case 0: return 1.e3f;
    case 1: return 1.f;
    case 2: return 1.e-3f;
    case 3: return 1.e-6f;
    default: return 1.f;
  }
}

int livox(const flb_preprocess_config& c, const flb_raw_layout& L, const unsigned char* r, int plsize, std::vector<Pt>& pl_surf) {
  std::vector<Pt> pl_full(plsize, Pt{0.f, 0.f, 0.f, 0.f, 0.f});   // pl_full.clear(); pl_full.resize(plsize)
  const double blind = c.blind;
  unsigned valid_num = 0;
  for (int i = 1; i < plsize; i++) {
    const unsigned char* rec = r + (size_t)i * L.stride;
    const unsigned line = field<uint8_t>(rec, L.off_line), tag = field<uint8_t>(rec, L.off_tag);
    if ((int)line < c.n_scans && ((tag & 0x30) == 0x10 || (tag & 0x30) == 0x00)) {
      valid_num++;
      if (valid_num % (unsigned)c.point_filter_num == 0) {
        pl_full[i].x = field<float>(rec, L.off_x);
        pl_full[i].y = field<float>(rec, L.off_y);
        pl_full[i].z = field<float>(rec, L.off_z);
        pl_full[i].intensity = field<uint8_t>(rec, L.off_intensity);
        pl_full[i].curvature = field<uint32_t>(rec, L.off_time) / float(1000000);
        if ((std::fabs(pl_full[i].x - pl_full[i - 1].x) > 1e-7) || (std::fabs(pl_full[i].y - pl_full[i - 1].y) > 1e-7) ||
            (std::fabs(pl_full[i].z - pl_full[i - 1].z) > 1e-7) &&
                (pl_full[i].x * pl_full[i].x + pl_full[i].y * pl_full[i].y + pl_full[i].z * pl_full[i].z > (blind * blind)))
          pl_surf.push_back(pl_full[i]);
      }
    }
  }
  return 0;
}

int ouster(const flb_preprocess_config& c, const flb_raw_layout& L, const unsigned char* r, int n, std::vector<Pt>& pl_surf) {
  const float scale = time_unit_scale(c.time_unit);
  const double blind = c.blind;
  for (int i = 0; i < n; i++) {
    if (i % c.point_filter_num != 0) continue;
    const unsigned char* rec = r + (size_t)i * L.stride;
    const float x = field<float>(rec, L.off_x), y = field<float>(rec, L.off_y), z = field<float>(rec, L.off_z);
    double range = x * x + y * y + z * z;
    if (range < (blind * blind)) continue;
    Pt p{x, y, z, field<float>(rec, L.off_intensity), 0.f};
    p.curvature = field<uint32_t>(rec, L.off_time) * scale;
    pl_surf.push_back(p);
  }
  return 0;
}

int velodyne(const flb_preprocess_config& c, const flb_raw_layout& L, const unsigned char* r, int plsize, std::vector<Pt>& pl_surf) {
  if (plsize == 0) return 0;
  const float scale = time_unit_scale(c.time_unit);
  const double blind = c.blind;
  const double omega_l = 0.361 * c.scan_rate;
  std::vector<bool> is_first(c.n_scans, true);
  std::vector<double> yaw_fp(c.n_scans, 0.0);
  std::vector<float> time_last(c.n_scans, 0.0);
  const bool given_offset_time = field<float>(r + (size_t)(plsize - 1) * L.stride, L.off_time) > 0;
  for (int i = 0; i < plsize; i++) {
    const unsigned char* rec = r + (size_t)i * L.stride;
    Pt p{field<float>(rec, L.off_x), field<float>(rec, L.off_y), field<float>(rec, L.off_z), field<float>(rec, L.off_intensity), 0.f};
    p.curvature = field<float>(rec, L.off_time) * scale;
    if (!given_offset_time) {
      const int layer = field<uint16_t>(rec, L.off_ring);
      if (layer >= c.n_scans) return 2;   // the reference indexes past its per-ring vectors here
      const double yaw_angle = std::atan2((double)p.y, (double)p.x) * 57.2957;
      if (is_first[layer]) {
        yaw_fp[layer] = yaw_angle;
        is_first[layer] = false;
        p.curvature = 0.0;
        time_last[layer] = p.curvature;
        continue;
      }
      if (yaw_angle <= yaw_fp[layer])
        p.curvature = (yaw_fp[layer] - yaw_angle) / omega_l;
      else
        p.curvature = (yaw_fp[layer] - yaw_angle + 360.0) / omega_l;
      if (p.curvature < time_last[layer]) p.curvature += 360.0 / omega_l;
      time_last[layer] = p.curvature;
    }
    if (i % c.point_filter_num == 0)
      if (p.x * p.x + p.y * p.y + p.z * p.z > (blind * blind)) pl_surf.push_back(p);
  }
  return 0;
}

}  // namespace

// Returns 0, 1 (bad arguments) or 2 (a Velodyne ring >= n_scans).  out_xyzi (n x 4) and out_curv (n) need room for n.
extern "C" int orc_preprocess(const flb_preprocess_config* cfg, const flb_raw_layout* layout, const void* records, int n,
                              float* out_xyzi, float* out_curv, int* n_out, float* last_curvature) {
  if (!cfg || !layout || n < 0 || (n > 0 && !records) || cfg->point_filter_num < 1 || cfg->n_scans < 1) return 1;
  const unsigned char* r = static_cast<const unsigned char*>(records);
  std::vector<Pt> pl_surf;
  int rc;
  switch (cfg->lidar_type) {
    case 1: rc = livox(*cfg, *layout, r, n, pl_surf); break;
    case 2: rc = velodyne(*cfg, *layout, r, n, pl_surf); break;
    case 3: rc = ouster(*cfg, *layout, r, n, pl_surf); break;
    default: return 1;
  }
  if (rc) return rc;
  for (size_t k = 0; k < pl_surf.size(); ++k) {
    out_xyzi[4 * k + 0] = pl_surf[k].x;
    out_xyzi[4 * k + 1] = pl_surf[k].y;
    out_xyzi[4 * k + 2] = pl_surf[k].z;
    out_xyzi[4 * k + 3] = pl_surf[k].intensity;
    out_curv[k] = pl_surf[k].curvature;
  }
  *n_out = (int)pl_surf.size();
  *last_curvature = pl_surf.empty() ? 0.f : pl_surf.back().curvature;
  return 0;
}
