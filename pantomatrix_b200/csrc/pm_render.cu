// SMPL-X mesh render (pantomatrix_b200/render.py): the frames of emage_utils/fast_render.py, one view per frame
// (render_one_sequence_no_gt) or two side by side (render_one_sequence_with_face, render_one_sequence).  Three launches
// per chunk of frames: pm_mesh_vertex_f32 (view transform, projection, snapping, vertex normals), pm_mesh_raster
// (visibility keys by atomicMin) and pm_mesh_shade_u8 (Lambert shading into the RGB frame), each taking the view count;
// plus pm_time_upsample_f32, the piecewise-linear frame-rate upsampling of the npz writer.  Contracts and the exact
// rules: include/pm_emage.h; CPU restatement: oracle/render_oracle.py.  Built with -fmad=false: every fp32 / fp64
// product and sum is rounded on its own, so the restatement reproduces the snapped coordinates and depths operation by
// operation.
#include <limits.h>
#include <math.h>

#include "pm_common.cuh"
#include "../../include/pm_emage.h"

namespace {

constexpr int W = 480, H = 720;           // one view (fast_render.py args, OffscreenRenderer(480, 720))
constexpr int SUB = 256;                  // 8 sub-pixel bits
constexpr float GUARD = 1048576.f;        // 2^20 pixels: |snapped| < 2^28, edge products < 2^59 fit int64
constexpr int BAD = INT_MIN;              // snapped x of a vertex that no triangle may use
// create_pose_camera(-2): rotation about x by -2 degrees, camera at (0, 1, 5), looking down its -z axis
constexpr float CAM_C = 0.99939082701909573f, CAM_S = -0.034899496702500969f, CAM_Y = 1.f, CAM_Z = 5.f;
// OrthographicCamera(xmag=1, ymag=1), pyrender's default znear / zfar; pyrender ignores the aspect ratio
constexpr float XMAG = 1.f, YMAG = 1.f, ZNEAR = 0.05f, ZFAR = 100.f;
// create_pose_light(-30): light travels along the pose's -z axis, so the direction toward the light is its +z axis
constexpr float LX = 0.f, LY = 0.5f, LZ = 0.86602540378443865f;
constexpr float COLOR = 220.f;            // uniform_color [220, 220, 220, 255]

struct ViewXf { float s0, ox0, oy0, oz0, s1, ox1, oy1, oz1; };

// The view's affine transform in fp32: p * scale, then + offset (the face view is v * 7 - (0, 10, 0)).
__device__ __forceinline__ float3 world(const float* v, int idx, float s, float ox, float oy, float oz) {
  const float* p = v + 3LL * idx;
  return make_float3(__fadd_rn(__fmul_rn(p[0], s), ox), __fadd_rn(__fmul_rn(p[1], s), oy),
                     __fadd_rn(__fmul_rn(p[2], s), oz));
}

// The one shading rule (swap it here and in oracle/render_oracle.py shade()): Lambert with the directional light,
// value = 220 max(0, n.l) rounded to nearest, the same for R, G and B.  n is normalised here; n = 0 shades black.
__device__ __forceinline__ unsigned char shade(float nx, float ny, float nz) {
  const float len = sqrtf(nx * nx + ny * ny + nz * nz);
  if (!(len > 0.f)) return 0;
  const float d = (nx * LX + ny * LY + nz * LZ) / len;
  return (unsigned char)min(255, __float2int_rn(COLOR * fmaxf(0.f, d)));
}

// NV views per frame (1 or 2): view k of frame f is image view k, read from verts_k.
template <int NV>
__global__ void __launch_bounds__(256) mesh_vertex_kernel(const float* __restrict__ v0, long long v0_fs,
                                                          const float* __restrict__ v1, long long v1_fs, int nv,
                                                          long long total, const ViewXf xf,
                                                          const int* __restrict__ faces,
                                                          const int* __restrict__ vf_ptr,
                                                          const int* __restrict__ vf_face, int2* __restrict__ xy,
                                                          float* __restrict__ depth, float* __restrict__ normal) {
  static_assert(NV == 1 || NV == 2, "one or two views per frame");
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long fv = i / nv;
  const int v = (int)(i % nv), view = (int)(fv & (NV - 1));
  const long long f = fv >> (NV - 1);
  const float* base = view ? v1 + f * v1_fs : v0 + f * v0_fs;
  const float s = view ? xf.s1 : xf.s0, ox = view ? xf.ox1 : xf.ox0, oy = view ? xf.oy1 : xf.oy0,
              oz = view ? xf.oz1 : xf.oz0;
  const float3 p = world(base, v, s, ox, oy, oz);
  // view transform (inverse camera pose), then the orthographic projection to pixels, row 0 at the top
  const float a = __fsub_rn(p.y, CAM_Y), b = __fsub_rn(p.z, CAM_Z);
  const float yv = __fadd_rn(__fmul_rn(CAM_C, a), __fmul_rn(CAM_S, b));
  const float zv = __fsub_rn(__fmul_rn(CAM_C, b), __fmul_rn(CAM_S, a));
  const float sx = __fmul_rn(__fadd_rn(__fdiv_rn(p.x, XMAG), 1.f), 0.5f * W);
  const float sy = __fmul_rn(__fsub_rn(1.f, __fdiv_rn(yv, YMAG)), 0.5f * H);
  const bool ok = fabsf(sx) <= GUARD && fabsf(sy) <= GUARD && isfinite(zv);   // NaN fails the comparisons
  xy[i] = ok ? make_int2(__float2int_rn(sx * SUB), __float2int_rn(sy * SUB)) : make_int2(BAD, BAD);
  depth[i] = -zv;

  // normal: sum of the unnormalised face normals over the incident faces in ascending face index, then normalised
  float nx = 0.f, ny = 0.f, nz = 0.f;
  for (int e = __ldg(vf_ptr + v), e1 = __ldg(vf_ptr + v + 1); e < e1; ++e) {
    const int t = __ldg(vf_face + e);
    const float3 A = world(base, __ldg(faces + 3 * t), s, ox, oy, oz);
    const float3 B = world(base, __ldg(faces + 3 * t + 1), s, ox, oy, oz);
    const float3 C = world(base, __ldg(faces + 3 * t + 2), s, ox, oy, oz);
    const float ux = B.x - A.x, uy = B.y - A.y, uz = B.z - A.z, wx = C.x - A.x, wy = C.y - A.y, wz = C.z - A.z;
    nx += uy * wz - uz * wy;
    ny += uz * wx - ux * wz;
    nz += ux * wy - uy * wx;
  }
  const float len = sqrtf(nx * nx + ny * ny + nz * nz);
  const float inv = len > 0.f ? 1.f / len : 0.f;
  float* n = normal + 3 * i;
  n[0] = nx * inv; n[1] = ny * inv; n[2] = nz * inv;
}

// A triangle in screen space, put in one winding (area2 > 0): its corner ids after the swap and snapped coordinates.
struct Tri { int id[3]; long long x[3], y[3], area2; };

__device__ __forceinline__ bool setup(const int2* __restrict__ xy, const int* __restrict__ faces, int t, Tri& T) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    T.id[k] = __ldg(faces + 3 * t + k);
    const int2 q = xy[T.id[k]];
    if (q.x == BAD) return false;
    T.x[k] = q.x; T.y[k] = q.y;
  }
  T.area2 = (T.x[1] - T.x[0]) * (T.y[2] - T.y[0]) - (T.y[1] - T.y[0]) * (T.x[2] - T.x[0]);
  if (T.area2 == 0) return false;
  if (T.area2 < 0) {                       // both sides are drawn: swap corners 1 and 2
    int ti = T.id[1]; T.id[1] = T.id[2]; T.id[2] = ti;
    long long tx = T.x[1]; T.x[1] = T.x[2]; T.x[2] = tx;
    long long ty = T.y[1]; T.y[1] = T.y[2]; T.y[2] = ty;
    T.area2 = -T.area2;
  }
  return true;
}

// Edge k runs from corner k+1 to corner k+2; its edge function is corner k's weight:
// w_k(c) = dx (c.y - y_{k+1}) - dy (c.x - x_{k+1}).
__device__ __forceinline__ long long edge(const Tri& T, int k, long long cx, long long cy) {
  const int p = (k + 1) % 3, q = (k + 2) % 3;
  return (T.x[q] - T.x[p]) * (cy - T.y[p]) - (T.y[q] - T.y[p]) * (cx - T.x[p]);
}

__global__ void __launch_bounds__(256) mesh_raster_kernel(const int2* __restrict__ xy, const float* __restrict__ depth,
                                                          int nv, const int* __restrict__ faces, int nf,
                                                          long long total, unsigned long long* __restrict__ vis) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long fv = i / nf;
  const int t = (int)(i % nf);
  Tri T;
  if (!setup(xy + fv * nv, faces, t, T)) return;
  const float* dp = depth + fv * nv;
  const double d0 = dp[T.id[0]], d1 = dp[T.id[1]], d2 = dp[T.id[2]];
  // pixels whose centre (p * 256 + 128) lies in the bounding box, clamped to the viewport
  const long long x0 = min(T.x[0], min(T.x[1], T.x[2])), x1 = max(T.x[0], max(T.x[1], T.x[2]));
  const long long y0 = min(T.y[0], min(T.y[1], T.y[2])), y1 = max(T.y[0], max(T.y[1], T.y[2]));
  const int px0 = (int)max(0LL, -((SUB / 2 - x0) >> 8)), px1 = (int)min((long long)W - 1, (x1 - SUB / 2) >> 8);
  const int py0 = (int)max(0LL, -((SUB / 2 - y0) >> 8)), py1 = (int)min((long long)H - 1, (y1 - SUB / 2) >> 8);
  if (px0 > px1 || py0 > py1) return;
  // top-left rule: a pixel centre on an edge belongs to the triangle whose inward normal (-dy, dx) points right, or
  // straight down for a horizontal edge: included edges test w >= 0, the others w > 0
  long long bias[3], stepx[3], stepy[3], row[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int p = (k + 1) % 3, q = (k + 2) % 3;
    const long long dx = T.x[q] - T.x[p], dy = T.y[q] - T.y[p];
    bias[k] = (dy < 0 || (dy == 0 && dx > 0)) ? 0 : 1;
    stepx[k] = -dy * SUB;
    stepy[k] = dx * SUB;
    row[k] = edge(T, k, (long long)px0 * SUB + SUB / 2, (long long)py0 * SUB + SUB / 2);
  }
  const double area = (double)T.area2;
  unsigned long long* out = vis + fv * (long long)(W * H);
  for (int py = py0; py <= py1; ++py) {
    long long w0 = row[0], w1 = row[1], w2 = row[2];
    for (int px = px0; px <= px1; ++px) {
      if (w0 >= bias[0] && w1 >= bias[1] && w2 >= bias[2]) {
        // depth = ((w0 d0 + w1 d1) + w2 d2) / area2 in fp64, each operation rounded, then rounded to fp32
        const double z = __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn((double)w0, d0), __dmul_rn((double)w1, d1)),
                                             __dmul_rn((double)w2, d2)), area);
        const float zf = __double2float_rn(z);
        if (zf >= ZNEAR && zf <= ZFAR) {
          const unsigned long long key = ((unsigned long long)__float_as_uint(zf) << 32) | (unsigned)t;
          unsigned long long* dst = out + py * W + px;
          // keys only decrease, so a stale read can only send us to the atomic needlessly
          if (key < *(volatile unsigned long long*)dst) atomicMin(dst, key);
        }
      }
      w0 += stepx[0]; w1 += stepx[1]; w2 += stepx[2];
    }
    row[0] += stepy[0]; row[1] += stepy[1]; row[2] += stepy[2];
  }
}

template <int NV>
__global__ void __launch_bounds__(256) mesh_shade_kernel(const unsigned long long* __restrict__ vis,
                                                         const int2* __restrict__ xy,
                                                         const float* __restrict__ normal, int nv,
                                                         const int* __restrict__ faces, long long total,
                                                         unsigned char* __restrict__ out, long long out_fs) {
  static_assert(NV == 1 || NV == 2, "one or two views per frame");
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long fv = i / (W * H);
  const int pix = (int)(i % (W * H)), py = pix / W, px = pix % W, view = (int)(fv & (NV - 1));
  unsigned char* dst = out + (fv >> (NV - 1)) * out_fs + ((long long)py * (NV * W) + view * W + px) * 3;
  const unsigned long long key = vis[i];
  unsigned char c = 0;
  if (key != ~0ull) {
    Tri T;
    setup(xy + fv * nv, faces, (int)(key & 0xffffffffu), T);
    const long long cx = (long long)px * SUB + SUB / 2, cy = (long long)py * SUB + SUB / 2;
    const double area = (double)T.area2;
    const float b0 = (float)((double)edge(T, 0, cx, cy) / area), b1 = (float)((double)edge(T, 1, cx, cy) / area),
                b2 = (float)((double)edge(T, 2, cx, cy) / area);
    const float* n = normal + 3 * fv * nv;
    const float* n0 = n + 3 * T.id[0];
    const float* n1 = n + 3 * T.id[1];
    const float* n2 = n + 3 * T.id[2];
    c = shade(b0 * n0[0] + b1 * n1[0] + b2 * n2[0], b0 * n0[1] + b1 * n1[1] + b2 * n2[1],
              b0 * n0[2] + b1 * n1[2] + b2 * n2[2]);
  }
  dst[0] = c; dst[1] = c; dst[2] = c;
}

// out[b, j, c] = fp32(a + d * frac) of the two source frames around position pos_j = j * ((t-1) / (k t - 1)) (the
// last one t-1 exactly), as numpy's linspace and motion_io.time_upsample_numpy compute it in fp64; k = 1 copies.
__global__ void __launch_bounds__(256) time_upsample_kernel(const float* __restrict__ x, long long x_bs, long long x_ts,
                                                            int t, int ch, int k, long long total,
                                                            float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % ch);
  const long long row = i / ch;
  const int n = k * t, j = (int)(row % n);
  const float* src = x + (row / n) * x_bs + c;
  if (k == 1) {
    out[i] = src[(long long)j * x_ts];
    return;
  }
  // linspace(0, t-1, n): i * step with step = (t-1) / (n-1); step = 0 (t = 1) gives 0 everywhere
  const double step = __ddiv_rn((double)(t - 1), (double)(n - 1));
  const double pos = j == n - 1 ? (double)(t - 1) : __dmul_rn((double)j, step);
  const int lo = min(max((int)floor(pos), 0), max(t - 2, 0));
  const double frac = __dsub_rn(pos, (double)lo);
  const float a = src[(long long)lo * x_ts], b = src[(long long)min(lo + 1, t - 1) * x_ts];
  out[i] = __double2float_rn(__dadd_rn((double)a, __dmul_rn((double)__fsub_rn(b, a), frac)));
}

inline unsigned blocks(long long n) { return (unsigned)((n + 255) / 256); }

int launch_vertex(int views, const float* verts0, long long v0_fs, const float* verts1, long long v1_fs, int n_verts,
                  int frames, const ViewXf& xf, const int* faces, const int* vf_ptr, const int* vf_face, int* xy,
                  float* depth, float* normal, void* stream) {
  PM_REQUIRE(views == 1 || views == 2);
  PM_REQUIRE(verts0 && (views == 1 || verts1) && faces && vf_ptr && vf_face && xy && depth && normal);
  PM_REQUIRE(n_verts > 0 && frames >= 0 && v0_fs >= 3LL * n_verts && (views == 1 || v1_fs >= 3LL * n_verts));
  const long long total = (long long)frames * views * n_verts;
  if (total == 0) return PM_OK;
  PM_REQUIRE(total / 256 < 0x7fffffffLL);
  auto kernel = views == 2 ? mesh_vertex_kernel<2> : mesh_vertex_kernel<1>;
  kernel<<<blocks(total), 256, 0, (cudaStream_t)stream>>>(verts0, v0_fs, verts1, v1_fs, n_verts, total, xf, faces,
                                                          vf_ptr, vf_face, reinterpret_cast<int2*>(xy), depth, normal);
  PM_LAUNCH_CHECK();
}

int launch_raster(int views, const int* xy, const float* depth, int n_verts, const int* faces, int n_faces, int frames,
                  unsigned long long* vis, void* stream) {
  PM_REQUIRE(views == 1 || views == 2);
  PM_REQUIRE(xy && depth && faces && vis && n_verts > 0 && n_faces >= 0 && frames >= 0);
  // the raster does not depend on the layout: one image per (frame, view)
  const long long total = (long long)frames * views * n_faces;
  if (total == 0) return PM_OK;
  PM_REQUIRE(total / 256 < 0x7fffffffLL);
  mesh_raster_kernel<<<blocks(total), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const int2*>(xy), depth,
                                                                       n_verts, faces, n_faces, total, vis);
  PM_LAUNCH_CHECK();
}

int launch_shade(int views, const unsigned long long* vis, const int* xy, const float* normal, int n_verts,
                 const int* faces, int frames, unsigned char* out, long long out_fs, void* stream) {
  PM_REQUIRE(views == 1 || views == 2);
  PM_REQUIRE(vis && xy && normal && faces && out && n_verts > 0 && frames >= 0 && out_fs >= 3LL * views * W * H);
  const long long total = (long long)frames * views * W * H;
  if (total == 0) return PM_OK;
  auto kernel = views == 2 ? mesh_shade_kernel<2> : mesh_shade_kernel<1>;
  kernel<<<blocks(total), 256, 0, (cudaStream_t)stream>>>(vis, reinterpret_cast<const int2*>(xy), normal, n_verts,
                                                          faces, total, out, out_fs);
  PM_LAUNCH_CHECK();
}

}  // namespace

extern "C" int pm_mesh_vertex_f32(const float* verts0, long long v0_fs, const float* verts1, long long v1_fs,
                                  int n_verts, int frames, float scale0, float ox0, float oy0, float oz0,
                                  float scale1, float ox1, float oy1, float oz1, const int* faces,
                                  const int* vf_ptr, const int* vf_face, int* xy, float* depth, float* normal,
                                  int views, void* stream) {
  return launch_vertex(views, verts0, v0_fs, verts1, v1_fs, n_verts, frames,
                       ViewXf{scale0, ox0, oy0, oz0, scale1, ox1, oy1, oz1}, faces, vf_ptr, vf_face, xy, depth, normal,
                       stream);
}

extern "C" int pm_mesh_raster(const int* xy, const float* depth, int n_verts, const int* faces, int n_faces,
                              int frames, unsigned long long* vis, int views, void* stream) {
  return launch_raster(views, xy, depth, n_verts, faces, n_faces, frames, vis, stream);
}

extern "C" int pm_mesh_shade_u8(const unsigned long long* vis, const int* xy, const float* normal, int n_verts,
                                const int* faces, int frames, unsigned char* out, long long out_fs, int views,
                                void* stream) {
  return launch_shade(views, vis, xy, normal, n_verts, faces, frames, out, out_fs, stream);
}

extern "C" int pm_time_upsample_f32(const float* x, long long x_bs, long long x_ts, int batch, int t, int channels,
                                    int k, float* out, void* stream) {
  PM_REQUIRE(x && out && batch >= 0 && t > 0 && channels > 0 && k >= 1);
  PM_REQUIRE((long long)k * t <= 0x7fffffffLL);
  const long long total = (long long)batch * k * t * channels;
  if (total == 0) return PM_OK;
  PM_REQUIRE(total / 256 < 0x7fffffffLL);
  time_upsample_kernel<<<blocks(total), 256, 0, (cudaStream_t)stream>>>(x, x_bs, x_ts, t, channels, k, total, out);
  PM_LAUNCH_CHECK();
}
