// TEST INFRASTRUCTURE ONLY -- CPU restatement of the TSDF integration the reference
// delegates to Open3D.  Nothing in the product path may import, link or call this file.
//
// PARITY UNPINNED: the arithmetic lives in the third-party wheel open3d==0.17.0
// (pinned in /root/reference/requirements.txt:15; README.md:371 insists on that version).
// The wheel is not installed here, its source is not under /root/reference and there is
// no network, and the reference has no test that pins TSDF values.  Round 2 tried to obtain it in the
// dev container and on the GPU box (scripts/try_open3d.sh; transcripts profiles/r02_open3d_attempt_*.log:
// no index reachable, nothing in /opt/wheelhouse, and 0.17.0 has no cp312 wheel).  The pin is prepared:
// tests/golden/make_tsdf_golden.py runs the literal Open3D call sequence and writes fixtures that
// tests/test_oracle_tsdf.py::test_open3d_golden_voxel_values / tests/test_oracle_mesh.py consume; they
// skip until somebody with the wheel runs the script.  This file restates
// Open3D 0.17.0's published algorithm
//   cpp/open3d/pipelines/integration/ScalableTSDFVolume.cpp  (Integrate, OpenVolumeUnit,
//       LocateVolumeUnit, ExtractTriangleMesh; ctor defaults volume_unit_resolution=16,
//       depth_sampling_stride=4)
//   cpp/open3d/pipelines/integration/UniformTSDFVolume.cpp   (IntegrateWithDepthToCameraDistanceMultiplier)
//   cpp/open3d/geometry/RGBDImageFactory.cpp + ImageFactory.cpp (CreateFromColorAndDepth ->
//       ConvertDepthToFloatImage; CreateDepthToCameraDistanceMultiplierFloatImage)
//   cpp/open3d/geometry/PointCloudFactory.cpp (CreatePointCloudFromFloatDepthImage)
// from memory, anchored on the reference's own call sites:
//   gs2mesh_utils/tsdf_utils.py:53-56  ScalableTSDFVolume(voxel_length, sdf_trunc, RGB8)
//   gs2mesh_utils/tsdf_utils.py:88-93  RGBDImage.create_from_color_and_depth(..., depth_scale, depth_trunc, False)
//   gs2mesh_utils/tsdf_utils.py:106-107 PinholeCameraIntrinsic + volume.integrate(rgbd, intr, inv(extrinsic))
// Points where the restatement had to choose (flagged DOUBT below) are the fp32
// summation order of Eigen's 4x4 * 4x1 product and `sdf * (1/trunc)` vs `sdf / trunc`.
//
// Compiled with -ffp-contract=off: Open3D wheels target baseline x86-64 (no FMA).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <memory>
#include <unordered_map>
#include <unordered_set>
#include <vector>

namespace {

constexpr int kRes = 16;     // volume_unit_resolution default
constexpr int kStride = 4;   // depth_sampling_stride default
constexpr int kVox = kRes * kRes * kRes;

struct Key {
  int x, y, z;
  bool operator==(const Key& o) const { return x == o.x && y == o.y && z == o.z; }
};
struct KeyHash {
  size_t operator()(const Key& k) const {
    uint64_t h = (uint64_t)(uint32_t)k.x * 0x9E3779B97F4A7C15ull;
    h ^= ((uint64_t)(uint32_t)k.y + 0x7F4A7C15ull + (h << 6) + (h >> 2));
    h ^= ((uint64_t)(uint32_t)k.z + 0x9E3779B9ull + (h << 6) + (h >> 2));
    return (size_t)h;
  }
};

struct Unit {  // one UniformTSDFVolume of 16^3 voxels, index x*256 + y*16 + z
  Key idx;
  double origin[3];
  std::vector<float> tsdf, weight;
  std::vector<double> color;  // 3 per voxel (Open3D stores Eigen::Vector3d)
};

struct Volume {
  double voxel_length, sdf_trunc, unit_length;
  bool with_color;
  std::unordered_map<Key, std::unique_ptr<Unit>, KeyHash> units;
  std::vector<Unit*> order;  // creation order (deterministic export)
};

inline int floor_div(double p, double len) { return (int)std::floor(p / len); }

// Sensitivity switches for the two DOUBT points (tests/test_oracle_tsdf.py::test_doubt_sensitivity): how far the results
// move if Open3D's binary resolves them the other way.  0 = the restatement (what the CUDA path is bit-exact with).
//   bit 0: 4x4 * 4x1 summed pairwise, (a0 + a1) + (a2 + a3) -- Eigen's NON-vectorised fixed-size reduction; the restatement
//          follows the vectorised evaluator (res = c0*x; res += c1*y; res += c2*z; res += c3*w), which is what a default
//          x86-64 build of Eigen 3.4 instantiates for aligned Matrix4f * Vector4f
//   bit 1: sdf / trunc instead of sdf * (1 / trunc)
//   bit 2: the product contracted to fused multiply-adds (a wheel built with -mfma)
//   bit 3: colour kept as the fp32 running mean the CUDA kernel computes, (c*w + rgb) / (w + 1) with one rounding per
//          operation, instead of Open3D's fp64 colour (tests pin the kernel's colour bit for bit with it)
int g_variant = 0;

// UniformTSDFVolume::IntegrateWithDepthToCameraDistanceMultiplier for one 16^3 unit.
void integrate_unit(Unit& u, const Volume& vol, const float* depth, const uint8_t* rgb, const float* mult, int W,
                    int H, float fx, float fy, float cx, float cy, const float E[16]) {
  const float vl = (float)vol.voxel_length;
  const float half = vl * 0.5f;
  const float trunc = (float)vol.sdf_trunc;
  const float trunc_inv = 1.0f / trunc;
  const float sx = E[2] * vl, sy = E[6] * vl, sz = E[10] * vl;  // extrinsic_scaled(:,2)
  const float safe_w = W - 0.0001f, safe_h = H - 0.0001f;
  for (int x = 0; x < kRes; ++x) {
    for (int y = 0; y < kRes; ++y) {
      // float(half + vl*x + origin) is evaluated in double (origin_ is a Vector3d) then rounded.
      const float px = (float)((double)(half + vl * x) + u.origin[0]);
      const float py = (float)((double)(half + vl * y) + u.origin[1]);
      const float pz = (float)((double)half + u.origin[2]);
      // DOUBT: Eigen Matrix4f * Vector4f summation order; sequential column accumulation assumed.
      float cxm = ((E[0] * px + E[1] * py) + E[2] * pz) + E[3] * 1.f;
      float cym = ((E[4] * px + E[5] * py) + E[6] * pz) + E[7] * 1.f;
      float czm = ((E[8] * px + E[9] * py) + E[10] * pz) + E[11] * 1.f;
      if (g_variant & 1) {
        cxm = (E[0] * px + E[1] * py) + (E[2] * pz + E[3] * 1.f);
        cym = (E[4] * px + E[5] * py) + (E[6] * pz + E[7] * 1.f);
        czm = (E[8] * px + E[9] * py) + (E[10] * pz + E[11] * 1.f);
      } else if (g_variant & 4) {
        cxm = std::fmaf(E[3], 1.f, std::fmaf(E[2], pz, std::fmaf(E[1], py, E[0] * px)));
        cym = std::fmaf(E[7], 1.f, std::fmaf(E[6], pz, std::fmaf(E[5], py, E[4] * px)));
        czm = std::fmaf(E[11], 1.f, std::fmaf(E[10], pz, std::fmaf(E[9], py, E[8] * px)));
      }
      for (int z = 0; z < kRes; ++z, cxm += sx, cym += sy, czm += sz) {
        if (czm <= 0) continue;
        const float u_f = cxm * fx / czm + cx + 0.5f;
        const float v_f = cym * fy / czm + cy + 0.5f;
        if (!(u_f >= 0.0001f && u_f < safe_w && v_f >= 0.0001f && v_f < safe_h)) continue;
        const int ui = (int)u_f, vi = (int)v_f;
        const float d = depth[(size_t)vi * W + ui];
        if (d <= 0.0f) continue;
        const int ind = (x * kRes + y) * kRes + z;
        const float sdf = (d - czm) * mult[(size_t)vi * W + ui];
        if (sdf > -trunc) {
          const float t = std::min(1.0f, (g_variant & 2) ? sdf / trunc : sdf * trunc_inv);  // DOUBT: multiply by reciprocal
          const float w = u.weight[ind];
          u.tsdf[ind] = (u.tsdf[ind] * w + t) / (w + 1.0f);
          if (vol.with_color && rgb) {
            const uint8_t* c = rgb + 3 * ((size_t)vi * W + ui);
            for (int k = 0; k < 3; ++k) {
              double& col = u.color[3 * (size_t)ind + k];
              if (g_variant & 8)
                col = (double)(((float)col * w + (float)c[k]) / (w + 1.0f));
              else
                col = (col * w + (double)c[k]) / (w + 1.0f);
            }
          }
          u.weight[ind] = w + 1.0f;
        }
      }
    }
  }
}

}  // namespace

extern "C" {

void* orc_tsdf_create(double voxel_length, double sdf_trunc, int with_color) {
  Volume* v = new Volume();
  v->voxel_length = voxel_length;
  v->sdf_trunc = sdf_trunc;
  v->unit_length = voxel_length * kRes;
  v->with_color = with_color != 0;
  return v;
}

void orc_tsdf_destroy(void* h) { delete static_cast<Volume*>(h); }

void orc_tsdf_set_variant(int bits) { g_variant = bits; }  // sensitivity study only; 0 = the restatement

int64_t orc_tsdf_num_units(void* h) { return (int64_t)static_cast<Volume*>(h)->order.size(); }

// RGBDImage::CreateFromColorAndDepth -> Image::ConvertDepthToFloatImage (T0b):
// d /= (float)depth_scale; if (d >= depth_trunc) d = 0 (comparison in double).
void orc_depth_convert(const float* in, int64_t n, double depth_scale, double depth_trunc, float* out) {
  const float s = (float)depth_scale;
  for (int64_t i = 0; i < n; ++i) {
    float d = in[i] / s;
    if ((double)d >= depth_trunc) d = 0.0f;
    out[i] = d;
  }
}

// Image::CreateDepthToCameraDistanceMultiplierFloatImage
void orc_depth_multiplier(int W, int H, double fx, double fy, double cx, double cy, float* out) {
  const float ix = 1.0f / (float)fx, iy = 1.0f / (float)fy;
  const float px = (float)cx, py = (float)cy;
  std::vector<float> xx(W), yy(H);
  for (int j = 0; j < W; ++j) xx[j] = (j - px) * ix;
  for (int i = 0; i < H; ++i) yy[i] = (i - py) * iy;
  for (int i = 0; i < H; ++i)
    for (int j = 0; j < W; ++j) out[(size_t)i * W + j] = sqrtf(xx[j] * xx[j] + yy[i] * yy[i] + 1.0f);
}

// ScalableTSDFVolume::Integrate.  depth: float [H,W] already converted (orc_depth_convert),
// rgb: uint8 [H,W,3] or NULL, extrinsic: world->camera, row-major double[16].
// `threads` > 1 integrates the touched units in parallel (units are independent, so the
// result is identical to Open3D's serial-over-units order); returns #units touched.
int64_t orc_tsdf_integrate(void* h, const float* depth, const uint8_t* rgb, int W, int H, double fx, double fy,
                           double cx, double cy, const double* extrinsic, int threads) {
  Volume& vol = *static_cast<Volume*>(h);
  std::vector<float> mult((size_t)W * H);
  orc_depth_multiplier(W, H, fx, fy, cx, cy, mult.data());

  // camera_pose = extrinsic^-1 (general 4x4 inverse via Gauss-Jordan in double)
  double a[4][8];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) {
      a[r][c] = extrinsic[4 * r + c];
      a[r][4 + c] = r == c ? 1.0 : 0.0;
    }
  for (int c = 0; c < 4; ++c) {
    int piv = c;
    for (int r = c + 1; r < 4; ++r)
      if (std::fabs(a[r][c]) > std::fabs(a[piv][c])) piv = r;
    if (piv != c)
      for (int k = 0; k < 8; ++k) std::swap(a[c][k], a[piv][k]);
    double d = a[c][c];
    for (int k = 0; k < 8; ++k) a[c][k] /= d;
    for (int r = 0; r < 4; ++r)
      if (r != c) {
        double f = a[r][c];
        for (int k = 0; k < 8; ++k) a[r][k] -= f * a[c][k];
      }
  }
  double pose[4][4];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) pose[r][c] = a[r][4 + c];

  // PointCloud::CreateFromDepthImage(depth, intrinsic, extrinsic, 1000, 1000, stride=4):
  // float images skip the scale/trunc step; every stride-th pixel with d > 0.
  std::unordered_set<Key, KeyHash> touched;
  std::vector<Unit*> todo;
  for (int i = 0; i < H; i += kStride)
    for (int j = 0; j < W; j += kStride) {
      const float p = depth[(size_t)i * W + j];
      if (!(p > 0)) continue;
      const double z = (double)p;
      const double x = (j - cx) * z / fx;
      const double y = (i - cy) * z / fy;
      double wp[3];
      for (int r = 0; r < 3; ++r) wp[r] = pose[r][0] * x + pose[r][1] * y + pose[r][2] * z + pose[r][3];
      int lo[3], hi[3];
      for (int r = 0; r < 3; ++r) {
        lo[r] = floor_div(wp[r] - vol.sdf_trunc, vol.unit_length);
        hi[r] = floor_div(wp[r] + vol.sdf_trunc, vol.unit_length);
      }
      for (int bx = lo[0]; bx <= hi[0]; ++bx)
        for (int by = lo[1]; by <= hi[1]; ++by)
          for (int bz = lo[2]; bz <= hi[2]; ++bz) {
            Key k{bx, by, bz};
            if (!touched.insert(k).second) continue;
            auto& slot = vol.units[k];
            if (!slot) {  // OpenVolumeUnit
              slot.reset(new Unit());
              slot->idx = k;
              slot->origin[0] = bx * vol.unit_length;
              slot->origin[1] = by * vol.unit_length;
              slot->origin[2] = bz * vol.unit_length;
              slot->tsdf.assign(kVox, 0.0f);
              slot->weight.assign(kVox, 0.0f);
              if (vol.with_color) slot->color.assign(3 * (size_t)kVox, 0.0);
              vol.order.push_back(slot.get());
            }
            todo.push_back(slot.get());
          }
    }
  float E[16];
  for (int k = 0; k < 16; ++k) E[k] = (float)extrinsic[k];
  const float ffx = (float)fx, ffy = (float)fy, fcx = (float)cx, fcy = (float)cy;
  const int64_t n = (int64_t)todo.size();
#pragma omp parallel for schedule(dynamic, 4) num_threads(threads > 0 ? threads : 1)
  for (int64_t t = 0; t < n; ++t) integrate_unit(*todo[t], vol, depth, rgb, mult.data(), W, H, ffx, ffy, fcx, fcy, E);
  return n;
}

// Unit indices in creation order: out[3*i..3*i+2].
void orc_tsdf_unit_indices(void* h, int* out) {
  Volume& vol = *static_cast<Volume*>(h);
  for (size_t i = 0; i < vol.order.size(); ++i) {
    out[3 * i] = vol.order[i]->idx.x;
    out[3 * i + 1] = vol.order[i]->idx.y;
    out[3 * i + 2] = vol.order[i]->idx.z;
  }
}

// Copies unit `i`'s 4096 voxels (x*256+y*16+z order).  color_out (3 doubles/voxel) may be NULL.
void orc_tsdf_unit_data(void* h, int64_t i, float* tsdf_out, float* weight_out, double* color_out) {
  Volume& vol = *static_cast<Volume*>(h);
  const Unit& u = *vol.order[(size_t)i];
  std::memcpy(tsdf_out, u.tsdf.data(), sizeof(float) * kVox);
  std::memcpy(weight_out, u.weight.data(), sizeof(float) * kVox);
  if (color_out && vol.with_color) std::memcpy(color_out, u.color.data(), sizeof(double) * 3 * kVox);
}

// Dense window export in the brick layout the CUDA path uses: bricks ordered
// (bx,by,bz) row-major inside the window [b0, b0+nb), voxels x*256+y*16+z inside a brick,
// (tsdf, weight) interleaved.  Units outside the window are counted in the return value.
int64_t orc_tsdf_export_bricks(void* h, const int* b0, const int* nb, float* tsdf_weight, uint8_t* allocated) {
  Volume& vol = *static_cast<Volume*>(h);
  int64_t outside = 0;
  for (Unit* u : vol.order) {
    const int bx = u->idx.x - b0[0], by = u->idx.y - b0[1], bz = u->idx.z - b0[2];
    if (bx < 0 || by < 0 || bz < 0 || bx >= nb[0] || by >= nb[1] || bz >= nb[2]) {
      ++outside;
      continue;
    }
    const size_t brick = ((size_t)bx * nb[1] + by) * nb[2] + bz;
    if (allocated) allocated[brick] = 1;
    float* dst = tsdf_weight + brick * 2 * kVox;
    for (int v = 0; v < kVox; ++v) {
      dst[2 * v] = u->tsdf[v];
      dst[2 * v + 1] = u->weight[v];
    }
  }
  return outside;
}

}  // extern "C"
