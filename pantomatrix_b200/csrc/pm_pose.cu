// Pose composition (EmageVQModel.decode, M.py:135-188), global translation (M.py:195-205) and the motion
// representation of the body model (pm_motion_rep_f32).
// Compiled with -fmad=false: the rotation formulas follow the reference's operation order
// (P.py:6-104) with one rounding per operation, like the eager torch kernels they replace.
// Contracts: include/pm_emage.h.
#include "pm_common.cuh"
#include "../../include/pm_emage.h"

namespace {

// Which decoder owns each of the 55 SMPL-X joints (M.py:75-90,181) and its slot inside that decoder's
// output: part 0 = upper (13 joints), 1 = lower (9), 2 = hands (30), 3 = jaw (face[:6]), 4 = none (eyes).
__constant__ int8_t kJointPart[55] = {
    1, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 3, 4, 4,
    2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2};
__constant__ int8_t kJointSlot[55] = {
    0, 1, 2, 0, 3, 4, 1, 5, 6, 2, 7, 8, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 0, 0, 0,
    0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29};

__device__ __forceinline__ float sqrt_pos(float x) { return x > 0.f ? sqrtf(x) : 0.f; }          // P.py:10-14
__device__ __forceinline__ float sign_like(float a, float b) { return ((a < 0.f) != (b < 0.f)) ? -a : a; }  // P.py:6-8

__device__ __forceinline__ float sin_half_over_angle(float half, float ang) {                      // P.py:35-43
  return fabsf(ang) < 1e-6f ? 0.5f - (ang * ang) / 48.f : sinf(half) / ang;
}

// rot6d -> axis-angle, P.py:49-58 then 16-44
__device__ void rot6d_to_aa(const float d[6], float aa[3]) {
  float n1 = fmaxf(sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), 1e-12f);
  const float b1x = d[0] / n1, b1y = d[1] / n1, b1z = d[2] / n1;
  const float dot = b1x * d[3] + b1y * d[4] + b1z * d[5];
  float b2x = d[3] - dot * b1x, b2y = d[4] - dot * b1y, b2z = d[5] - dot * b1z;
  float n2 = fmaxf(sqrtf(b2x * b2x + b2y * b2y + b2z * b2z), 1e-12f);
  b2x /= n2; b2y /= n2; b2z /= n2;
  const float b3x = b1y * b2z - b1z * b2y;
  const float b3y = b1z * b2x - b1x * b2z;
  const float b3z = b1x * b2y - b1y * b2x;
  // matrix rows: (b1), (b2), (b3); m[i][j]
  const float m00 = b1x, m11 = b2y, m22 = b3z;
  const float w = 0.5f * sqrt_pos(1.f + m00 + m11 + m22);
  float x = 0.5f * sqrt_pos(1.f + m00 - m11 - m22);
  float y = 0.5f * sqrt_pos(1.f - m00 + m11 - m22);
  float z = 0.5f * sqrt_pos(1.f - m00 - m11 + m22);
  x = sign_like(x, b3y - b2z);     // m21 - m12
  y = sign_like(y, b1z - b3x);     // m02 - m20
  z = sign_like(z, b2x - b1y);     // m10 - m01
  const float n = sqrtf(x * x + y * y + z * z);
  const float half = atan2f(n, w);
  const float ang = 2.f * half;
  const float s = sin_half_over_angle(half, ang);
  aa[0] = x / s; aa[1] = y / s; aa[2] = z / s;
}

// axis-angle -> first two rows of the rotation matrix, P.py:63-104
__device__ void aa_to_rot6d(const float aa[3], float o[6]) {
  const float ang = sqrtf(aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2]);
  const float half = 0.5f * ang;
  const float s = sin_half_over_angle(half, ang);
  const float r = cosf(half), i = aa[0] * s, j = aa[1] * s, k = aa[2] * s;
  const float two_s = 2.0f / (r * r + i * i + j * j + k * k);
  o[0] = 1.f - two_s * (j * j + k * k);
  o[1] = two_s * (i * j - k * r);
  o[2] = two_s * (i * k + j * r);
  o[3] = two_s * (i * j + k * r);
  o[4] = 1.f - two_s * (i * i + k * k);
  o[5] = two_s * (j * k - i * r);
}

__global__ void __launch_bounds__(256) pose_compose_kernel(
    const float* __restrict__ face, const float* __restrict__ upper, const float* __restrict__ hands,
    const float* __restrict__ lower, float* __restrict__ expression, float* __restrict__ axis_angle,
    float* __restrict__ motion4inf, long long bt) {
  const long long total = bt * 64;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i >> 6;
    const int w = (int)(i & 63);
    if (w < 55) {
      const int part = kJointPart[w], slot = kJointSlot[w];
      const float* src = nullptr;
      if (part == 0 && upper) src = upper + r * 78 + slot * 6;
      else if (part == 1 && lower) src = lower + r * 61 + slot * 6;
      else if (part == 2 && hands) src = hands + r * 180 + slot * 6;
      else if (part == 3 && face) src = face + r * 106;
      float aa[3] = {0.f, 0.f, 0.f};
      if (src) {
        float d[6];
#pragma unroll
        for (int c = 0; c < 6; ++c) d[c] = src[c];
        rot6d_to_aa(d, aa);
      }
      float o[6];
      aa_to_rot6d(aa, o);
#pragma unroll
      for (int c = 0; c < 3; ++c) axis_angle[r * 165 + w * 3 + c] = aa[c];
#pragma unroll
      for (int c = 0; c < 6; ++c) motion4inf[r * 337 + w * 6 + c] = o[c];
    } else if (w == 55) {
#pragma unroll
      for (int c = 0; c < 7; ++c) motion4inf[r * 337 + 330 + c] = lower ? lower[r * 61 + 54 + c] : 0.f;
    } else {
      for (int c = w - 56; c < 100; c += 8) expression[r * 100 + c] = face ? face[r * 106 + 6 + c] : 0.f;
    }
  }
}

__global__ void __launch_bounds__(64) global_trans_kernel(const float* __restrict__ rec, int ld, int vel_off,
                                                          const float* __restrict__ ref_trans, int ref_bs, float dt,
                                                          float* __restrict__ trans, int t) {
  const int b = blockIdx.x;
  const float* __restrict__ v = rec + (long long)b * t * ld + vel_off;
  float* __restrict__ o = trans + (long long)b * t * 3;
  if (threadIdx.x < 2) {                          // x (axis 0) and z (axis 2): sequential, reference order
    const int ax = threadIdx.x * 2;
    float pos = ref_trans[(long long)b * ref_bs + ax];
    o[ax] = pos;
    for (int i = 1; i < t; ++i) {
      pos = v[(long long)(i - 1) * ld + ax] * dt + pos;     // one rounding per op (-fmad=false)
      o[(long long)i * 3 + ax] = pos;
    }
  } else {
    for (int i = threadIdx.x - 2; i < t; i += blockDim.x - 2) o[(long long)i * 3 + 1] = v[(long long)i * ld + 1];
  }
}

// rot6d rows of the selected joints -> axis-angle of all 55 joints (zeros elsewhere): rotation_6d_to_axis_angle +
// recover_from_mask_ts of the CaMN / DisCo heads (camn:274-277).  slot[j] = position of joint j among the selected
// joints, or -1.
__global__ void __launch_bounds__(256) rot6d_to_aa_kernel(const float* __restrict__ rot6d, long long rows, int n_sel,
                                                          const int* __restrict__ slot, float* __restrict__ out) {
  const long long total = rows * 55;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / 55;
    const int j = (int)(i % 55);
    const int sl = slot[j];
    float aa[3] = {0.f, 0.f, 0.f};
    if (sl >= 0) {
      float d[6];
#pragma unroll
      for (int c = 0; c < 6; ++c) d[c] = rot6d[(r * n_sel + sl) * 6 + c];
      rot6d_to_aa(d, aa);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) out[r * 165 + j * 3 + c] = aa[c];
  }
}

// DisCo content mix (disco:250-251): w = softmax(sel, 2 logits); out = w0 * c1 + w1 * c2, one rounding per op
__global__ void __launch_bounds__(256) softmax2_mix_kernel(const float* __restrict__ sel, const float* __restrict__ c1,
                                                           const float* __restrict__ c2, float* __restrict__ out,
                                                           long long rows, int ch, int ldo) {
  const long long total = rows * ch;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / ch;
    const int c = (int)(i % ch);
    const float a = sel[2 * r], b = sel[2 * r + 1];
    const float m = fmaxf(a, b);
    const float ea = expf(a - m), eb = expf(b - m);
    const float s = ea + eb;
    out[r * ldo + c] = (ea / s) * c1[i] + (eb / s) * c2[i];
  }
}

// get_motion_rep_tensor (emage_utils/motion_rep_transfer.py:31-72): per (frame, joint) the 15 values
// [position | velocity | rot6d | angular velocity].  Differences are one-sided at both ends of a clip and central inside,
// subtracted and then divided by dt or 2 dt (float32 roundings of the reference's Python scalars), one rounding per op.
__global__ void __launch_bounds__(256) motion_rep_kernel(const float* __restrict__ poses, long long pose_bs,
                                                         long long pose_ts, const float* __restrict__ joints,
                                                         long long rows, int t, float dt, float two_dt,
                                                         float* __restrict__ rep) {
  const long long total = rows * 55;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / 55;
    const int j = (int)(i % 55);
    const long long b = r / t;
    const int tt = (int)(r % t);
    const int hi = tt + 1 < t ? tt + 1 : tt, lo = tt > 0 ? tt - 1 : tt;
    const float den = (tt == 0 || tt == t - 1) ? dt : two_dt;
    const float* jh = joints + ((b * t + hi) * 55 + j) * 3;
    const float* jl = joints + ((b * t + lo) * 55 + j) * 3;
    const float* p = poses + b * pose_bs + (long long)tt * pose_ts + 3 * j;
    const float* ph = poses + b * pose_bs + (long long)hi * pose_ts + 3 * j;
    const float* pl = poses + b * pose_bs + (long long)lo * pose_ts + 3 * j;
    float* o = rep + r * 825 + j * 15;
    const float aa[3] = {p[0], p[1], p[2]};
    float r6[6];
    aa_to_rot6d(aa, r6);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      o[c] = joints[(r * 55 + j) * 3 + c];
      o[3 + c] = (jh[c] - jl[c]) / den;
      o[12 + c] = (ph[c] - pl[c]) / den;
    }
#pragma unroll
    for (int c = 0; c < 6; ++c) o[6 + c] = r6[c];
  }
}

}  // namespace

extern "C" int pm_motion_rep_f32(const float* poses, long long pose_bs, long long pose_ts, const float* joints,
                                 int batch, int t, float dt, float two_dt, float* rep15d, void* stream) {
  PM_REQUIRE(poses && joints && rep15d && batch >= 0 && t >= 2 && dt > 0.f && two_dt > 0.f);
  const long long rows = (long long)batch * t;
  if (rows == 0) return PM_OK;
  long long g = (rows * 55 + 255) / 256;
  if (g > 148 * 16) g = 148 * 16;
  motion_rep_kernel<<<(unsigned)g, 256, 0, (cudaStream_t)stream>>>(poses, pose_bs, pose_ts, joints, rows, t, dt, two_dt,
                                                                  rep15d);
  PM_LAUNCH_CHECK();
}

extern "C" int pm_rot6d_to_aa_f32(const float* rot6d, long long rows, int n_sel, const int* slot, float* out, void* stream) {
  PM_REQUIRE(rot6d && slot && out && rows >= 0 && n_sel > 0 && n_sel <= 55);
  if (rows == 0) return PM_OK;
  long long g = (rows * 55 + 255) / 256;
  if (g > 148 * 16) g = 148 * 16;
  rot6d_to_aa_kernel<<<(unsigned)g, 256, 0, (cudaStream_t)stream>>>(rot6d, rows, n_sel, slot, out);
  PM_LAUNCH_CHECK();
}

extern "C" int pm_softmax2_mix_f32(const float* sel, const float* c1, const float* c2, float* out, long long rows,
                                   int ch, int ldo, void* stream) {
  PM_REQUIRE(sel && c1 && c2 && out && rows >= 0 && ch > 0 && ldo >= ch);
  if (rows == 0) return PM_OK;
  long long g = (rows * ch + 255) / 256;
  if (g > 148 * 16) g = 148 * 16;
  softmax2_mix_kernel<<<(unsigned)g, 256, 0, (cudaStream_t)stream>>>(sel, c1, c2, out, rows, ch, ldo);
  PM_LAUNCH_CHECK();
}

extern "C" int pm_pose_compose_f32(const float* face, const float* upper, const float* hands, const float* lower,
                                   float* expression, float* axis_angle, float* motion4inf, long long bt,
                                   void* stream) {
  PM_REQUIRE(expression && axis_angle && motion4inf && bt >= 0);
  if (bt == 0) return PM_OK;
  long long g = (bt * 64 + 255) / 256;
  if (g > 148 * 16) g = 148 * 16;
  pose_compose_kernel<<<(unsigned)g, 256, 0, (cudaStream_t)stream>>>(face, upper, hands, lower, expression,
                                                                    axis_angle, motion4inf, bt);
  PM_LAUNCH_CHECK();
}

extern "C" int pm_global_trans_f32(const float* rec, int ld, int vel_off, const float* ref_trans, int ref_bs, float dt,
                                   float* trans, int batch, int t, void* stream) {
  PM_REQUIRE(rec && ref_trans && trans && batch >= 0 && t >= 0 && ld >= vel_off + 3 && ref_bs >= 0);
  if (batch == 0 || t == 0) return PM_OK;
  global_trans_kernel<<<batch, 64, 0, (cudaStream_t)stream>>>(rec, ld, vel_off, ref_trans, ref_bs, dt, trans, t);
  PM_LAUNCH_CHECK();
}
