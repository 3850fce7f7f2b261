// SMPL-X body model (pantomatrix_b200/body_model.py): rest joints + Rodrigues + forward kinematics in one launch
// (pm_smplx_fk_f32) and linear blend skinning (pm_smplx_skin_f32).  The vertex blend GEMM between the two is the
// tap-GEMM (pm_tapgemm_tc / pm_tapgemm_f32), whose A operand the FK kernel writes.  Contracts: include/pm_emage.h.
#include "pm_common.cuh"
#include "../../include/pm_emage.h"

namespace {

constexpr int NJ = 55;                  // SMPL-X joints
constexpr int NJ3 = NJ * 3;
constexpr int NB = 300, NE = 100;       // shape / expression coefficients
constexpr int NC = NB + NE;             // blend coefficients per frame
constexpr int FK_F = 16;                // frames per CTA: every j_dirs element read from L2 serves 16 frames
constexpr int FK_THREADS = 256;
constexpr size_t FK_SMEM = sizeof(float) * FK_F * (NC + NJ3 + NJ * 12);

struct FkArgs {
  const float* poses; long long pose_bs, pose_ts;
  const float* betas; long long b_bs;
  const float* expr; long long e_bs, e_ts;
  const float* transl; long long t_bs, t_ts;
  unsigned long long mask;
  int t;
  long long rows;
  const float* j_template; const float* j_dirs; const float* pose_mean;
  const int* parents; const int* order; const int* level_start; int n_levels;
  float* joints; float* rel; float* feat; int ld_feat;
  PmPlanes P;
};

template <bool F16>
__device__ __forceinline__ void put_feat(const FkArgs& a, long long row, int c, float v) {
  if (a.feat) a.feat[row * a.ld_feat + c] = v;
  if (a.P.ptr) pm_store_planes_t<F16>(a.P, row, c, v);
}

template <bool F16>
__global__ void __launch_bounds__(FK_THREADS) smplx_fk_kernel(const FkArgs a) {
  extern __shared__ float sm[];
  float* coef = sm;                       // [FK_F][NC]  betas | expression of each frame
  float* J = coef + FK_F * NC;            // [FK_F][NJ3] rest joints
  float* G = J + FK_F * NJ3;              // [FK_F][NJ][12]: R (9, row-major), then the global 3x4 transform
  const int tid = threadIdx.x;
  const long long r0 = (long long)blockIdx.x * FK_F;
  const int nf = (int)min((long long)FK_F, a.rows - r0);
  const bool want_feat = a.feat || a.P.ptr;

  // 1. blend coefficients -> shared memory and A-operand columns [0, 400)
  for (int i = tid; i < nf * NC; i += FK_THREADS) {
    const int f = i / NC, k = i % NC;
    const long long r = r0 + f, b = r / a.t, tt = r % a.t;
    float v = 0.f;
    if (k < NB) {
      if (a.betas) v = a.betas[b * a.b_bs + k];
    } else if (a.expr) {
      v = a.expr[b * a.e_bs + tt * a.e_ts + (k - NB)];
    }
    coef[i] = v;
    if (want_feat) put_feat<F16>(a, r, k, v);
  }

  // 2. Rodrigues per (frame, joint) (smplx batch_rodrigues: angle = |r + 1e-8|, R = I + sin K + (1 - cos) K K);
  //    pose feature R - I of joints 1..54 -> A-operand columns [400, 886)
  for (int i = tid; i < nf * NJ; i += FK_THREADS) {
    const int f = i / NJ, j = i % NJ;
    const long long r = r0 + f, b = r / a.t, tt = r % a.t;
    const float* p = a.poses + b * a.pose_bs + tt * a.pose_ts + 3 * j;
    const bool use = (a.mask >> j) & 1ull;
    const float rx = (use ? p[0] : 0.f) + a.pose_mean[3 * j];
    const float ry = (use ? p[1] : 0.f) + a.pose_mean[3 * j + 1];
    const float rz = (use ? p[2] : 0.f) + a.pose_mean[3 * j + 2];
    const float ex = rx + 1e-8f, ey = ry + 1e-8f, ez = rz + 1e-8f;
    const float ang = sqrtf(ex * ex + ey * ey + ez * ez);
    const float kx = rx / ang, ky = ry / ang, kz = rz / ang;
    float s, c;
    sincosf(ang, &s, &c);
    const float omc = 1.f - c;
    float R[9];
    R[0] = 1.f + omc * (-kz * kz - ky * ky);
    R[1] = -s * kz + omc * (kx * ky);
    R[2] = s * ky + omc * (kx * kz);
    R[3] = s * kz + omc * (kx * ky);
    R[4] = 1.f + omc * (-kz * kz - kx * kx);
    R[5] = -s * kx + omc * (ky * kz);
    R[6] = -s * ky + omc * (kx * kz);
    R[7] = s * kx + omc * (ky * kz);
    R[8] = 1.f + omc * (-ky * ky - kx * kx);
    float* g = G + (f * NJ + j) * 12;
#pragma unroll
    for (int m = 0; m < 9; ++m) g[m] = R[m];
    if (want_feat && j > 0) {
#pragma unroll
      for (int m = 0; m < 9; ++m) put_feat<F16>(a, r, NC + (j - 1) * 9 + m, (m % 4 == 0) ? R[m] - 1.f : R[m]);
    }
  }
  __syncthreads();

  // 3. rest joints J = j_template + j_dirs^T [betas | expression]: one output coordinate per thread, all frames of the
  //    CTA at once (each j_dirs element is loaded once per 16 frames; the coefficients are shared-memory broadcasts)
  if (tid < NJ3) {
    float acc[FK_F];
    const float base = a.j_template[tid];
#pragma unroll
    for (int f = 0; f < FK_F; ++f) acc[f] = base;
    const int k0 = a.betas ? 0 : NB, k1 = a.expr ? NC : NB;
#pragma unroll 2
    for (int k = k0; k < k1; ++k) {
      const float w = __ldg(a.j_dirs + (long long)k * NJ3 + tid);
#pragma unroll
      for (int f = 0; f < FK_F; ++f) acc[f] = fmaf(w, coef[f * NC + k], acc[f]);
    }
#pragma unroll
    for (int f = 0; f < FK_F; ++f)
      if (f < nf) J[f * NJ3 + tid] = acc[f];
  }
  __syncthreads();

  // 4. forward kinematics, one tree level per step: G_j = G_parent [R_j | J_j - J_parent]
  for (int l = 0; l < a.n_levels; ++l) {
    const int s0 = a.level_start[l], n = a.level_start[l + 1] - s0;
    for (int i = tid; i < nf * n; i += FK_THREADS) {
      const int f = i / n, j = a.order[s0 + i % n], pj = a.parents[j];
      float* g = G + (f * NJ + j) * 12;
      const float* Jf = J + f * NJ3;
      float R[9];
#pragma unroll
      for (int m = 0; m < 9; ++m) R[m] = g[m];
      float o[12];
      if (pj < 0) {
#pragma unroll
        for (int row = 0; row < 3; ++row) {
          o[row * 4] = R[row * 3]; o[row * 4 + 1] = R[row * 3 + 1]; o[row * 4 + 2] = R[row * 3 + 2];
          o[row * 4 + 3] = Jf[3 * j + row];
        }
      } else {
        const float t0 = Jf[3 * j] - Jf[3 * pj], t1 = Jf[3 * j + 1] - Jf[3 * pj + 1], t2 = Jf[3 * j + 2] - Jf[3 * pj + 2];
        const float* gp = G + (f * NJ + pj) * 12;
#pragma unroll
        for (int row = 0; row < 3; ++row) {
          const float p0 = gp[row * 4], p1 = gp[row * 4 + 1], p2 = gp[row * 4 + 2];
#pragma unroll
          for (int c = 0; c < 3; ++c) o[row * 4 + c] = p0 * R[c] + p1 * R[3 + c] + p2 * R[6 + c];
          o[row * 4 + 3] = p0 * t0 + p1 * t1 + p2 * t2 + gp[row * 4 + 3];
        }
      }
#pragma unroll
      for (int m = 0; m < 12; ++m) g[m] = o[m];
    }
    __syncthreads();
  }

  // 5. posed joints (+ transl) and, when vertices are wanted, the relative transforms A_j = G_j - [0 | G_j (J_j, 0)]
  for (int i = tid; i < nf * NJ3; i += FK_THREADS) {
    const int f = i / NJ3, e = i % NJ3, j = e / 3, c = e % 3;
    const long long r = r0 + f;
    float v = G[(f * NJ + j) * 12 + c * 4 + 3];
    if (a.transl) v += a.transl[(r / a.t) * a.t_bs + (r % a.t) * a.t_ts + c];
    a.joints[r0 * NJ3 + i] = v;
  }
  if (a.rel) {
    for (int i = tid; i < nf * NJ * 12; i += FK_THREADS) {
      const int f = i / (NJ * 12), e = i % (NJ * 12), j = e / 12, m = e % 12;
      const float* g = G + (f * NJ + j) * 12;
      float v = g[m];
      if ((m & 3) == 3) {
        const float* Jj = J + f * NJ3 + 3 * j;
        const int row = m >> 2;
        v = g[m] - (g[row * 4] * Jj[0] + g[row * 4 + 1] * Jj[1] + g[row * 4 + 2] * Jj[2]);
      }
      a.rel[r0 * NJ * 12 + i] = v;
    }
  }
}

// One CTA per frame: the frame's 55 relative transforms are staged in shared memory, each thread skins vertices
// v, v + 256, ... in place: x <- (sum_j w_vj A_j) (x, 1) + transl.
__global__ void __launch_bounds__(256) smplx_skin_kernel(float* __restrict__ verts, long long ld, int nv,
                                                         const int* __restrict__ row_ptr, const int* __restrict__ col,
                                                         const float* __restrict__ val, const float* __restrict__ rel,
                                                         const float* __restrict__ transl, long long t_bs, long long t_ts,
                                                         int t) {
  __shared__ float A[NJ * 12];
  const long long r = blockIdx.x;
  for (int i = threadIdx.x; i < NJ * 12; i += blockDim.x) A[i] = rel[r * NJ * 12 + i];
  float d[3] = {0.f, 0.f, 0.f};
  if (transl) {
    const float* tr = transl + (r / t) * t_bs + (r % t) * t_ts;
    d[0] = tr[0]; d[1] = tr[1]; d[2] = tr[2];
  }
  __syncthreads();
  float* __restrict__ row = verts + r * ld;
  for (int v = threadIdx.x; v < nv; v += blockDim.x) {
    // the HBM loads first, so they are in flight during the dependent (L2-resident) CSR reads
    const float x = row[3 * v], y = row[3 * v + 1], z = row[3 * v + 2];
    float T[12];
#pragma unroll
    for (int m = 0; m < 12; ++m) T[m] = 0.f;
    const int e0 = __ldg(row_ptr + v), e1 = __ldg(row_ptr + v + 1);
#pragma unroll 4
    for (int e = e0; e < e1; ++e) {
      const float w = __ldg(val + e);
      const float* Aj = A + __ldg(col + e) * 12;
#pragma unroll
      for (int m = 0; m < 12; ++m) T[m] = fmaf(w, Aj[m], T[m]);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) row[3 * v + c] = T[c * 4] * x + T[c * 4 + 1] * y + T[c * 4 + 2] * z + T[c * 4 + 3] + d[c];
  }
}

template <bool F16>
int launch_fk(const FkArgs& a, cudaStream_t st) {
  static unsigned long long configured = 0;
  if (pm_first_use_on_device(configured)) {
    const cudaError_t e = cudaFuncSetAttribute(smplx_fk_kernel<F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FK_SMEM);
    if (e != cudaSuccess) return (int)e;
  }
  smplx_fk_kernel<F16><<<(unsigned)((a.rows + FK_F - 1) / FK_F), FK_THREADS, FK_SMEM, st>>>(a);
  PM_LAUNCH_CHECK();
}

}  // namespace

extern "C" int pm_smplx_fk_f32(const float* poses, long long pose_bs, long long pose_ts,
                               const float* betas, long long b_bs,
                               const float* expr, long long e_bs, long long e_ts,
                               const float* transl, long long t_bs, long long t_ts,
                               long long joint_mask, int batch, int t,
                               const float* j_template, const float* j_dirs, const float* pose_mean,
                               const int* parents, const int* level_order, const int* level_start, int n_levels,
                               float* joints, float* rel_transforms, float* feat, int ld_feat,
                               uint16_t* planes, long long p_ps, int p_ld, int p_nsplit, void* stream) {
  PM_TAKE_FMT(p_nsplit, f16);
  PM_REQUIRE(poses && j_template && j_dirs && pose_mean && parents && level_order && level_start && joints);
  PM_REQUIRE(batch >= 0 && t >= 0 && n_levels >= 1 && n_levels <= NJ);
  PM_REQUIRE(!feat || ld_feat >= NC + 486);
  PM_REQUIRE(pm_planes_ok(planes, p_ps, p_ld, p_nsplit, NC + 486, false));
  const long long rows = (long long)batch * t;
  if (rows == 0) return PM_OK;
  FkArgs a{poses, pose_bs, pose_ts, betas, b_bs, expr, e_bs, e_ts, transl, t_bs, t_ts,
           (unsigned long long)joint_mask, t, rows, j_template, j_dirs, pose_mean,
           parents, level_order, level_start, n_levels, joints, rel_transforms, feat, ld_feat,
           PmPlanes{reinterpret_cast<__nv_bfloat16*>(planes), p_ps, p_ld, p_nsplit}};
  const cudaStream_t st = (cudaStream_t)stream;
  return f16 ? launch_fk<true>(a, st) : launch_fk<false>(a, st);
}

extern "C" int pm_smplx_skin_f32(float* verts, long long ld, long long rows, int n_verts,
                                 const int* row_ptr, const int* col, const float* val, const float* rel_transforms,
                                 const float* transl, long long t_bs, long long t_ts, int t, void* stream) {
  PM_REQUIRE(verts && row_ptr && col && val && rel_transforms && rows >= 0 && n_verts > 0 && ld >= 3LL * n_verts);
  PM_REQUIRE(!transl || t > 0);
  if (rows == 0) return PM_OK;
  PM_REQUIRE(rows <= 0x7fffffffLL);
  smplx_skin_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(verts, ld, n_verts, row_ptr, col, val,
                                                                      rel_transforms, transl, t_bs, t_ts, t > 0 ? t : 1);
  PM_LAUNCH_CHECK();
}
