// Per-pose similarity Procrustes (common/loss.py:34-66) in Horn's quaternion form, fp64, for
// pose_loss.cu's P-MPJPE (the metric and the differentiable loss).
// H = X0^T Y0 of the centred, normalised target X0 and prediction Y0.  The symmetric 4x4 N(H)
// (Horn 1987) has as its largest eigenvalue the reference's optimal trace s1 + s2 + sign(det H) s3
// of the SVD, and as its eigenvector the unit quaternion of the rotation.  The eigen-decomposition
// is cyclic Jacobi; all four eigenpairs come out of the sweeps (the loss's backward needs them).
#pragma once

namespace vp3d {
namespace {

constexpr int kJacobiSweeps = 12;

// One Jacobi rotation zeroing A[p][q] of the symmetric 4x4 A, accumulated into the columns of V.
template <int p, int q>
__device__ __forceinline__ void jacobi_rotate(double (&A)[4][4], double (&V)[4][4]) {
  const double apq = A[p][q];
  if (apq == 0.0) return;
  const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
  const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
  const double c = rsqrt(t * t + 1.0), s = t * c;
#pragma unroll
  for (int k = 0; k < 4; ++k) {  // A <- A J (columns p, q)
    const double akp = A[k][p], akq = A[k][q];
    A[k][p] = c * akp - s * akq;
    A[k][q] = s * akp + c * akq;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {  // A <- J^T A (rows p, q)
    const double apk = A[p][k], aqk = A[q][k];
    A[p][k] = c * apk - s * aqk;
    A[q][k] = s * apk + c * aqk;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double vkp = V[k][p], vkq = V[k][q];
    V[k][p] = c * vkp - s * vkq;
    V[k][q] = s * vkp + c * vkq;
  }
}

// Eigen-decomposition of N(H): on return A's diagonal holds the eigenvalues (unsorted) and column k
// of V the unit eigenvector of A[k][k].
__device__ __forceinline__ void horn_eigen(const double (&H)[3][3], double (&A)[4][4], double (&V)[4][4]) {
  // S = H^T: S_ab = sum_j y_a x_b (Horn 1987, eq. for N)
  const double Sxx = H[0][0], Sxy = H[1][0], Sxz = H[2][0];
  const double Syx = H[0][1], Syy = H[1][1], Syz = H[2][1];
  const double Szx = H[0][2], Szy = H[1][2], Szz = H[2][2];
  A[0][0] = Sxx + Syy + Szz; A[0][1] = Syz - Szy; A[0][2] = Szx - Sxz; A[0][3] = Sxy - Syx;
  A[1][0] = Syz - Szy; A[1][1] = Sxx - Syy - Szz; A[1][2] = Sxy + Syx; A[1][3] = Szx + Sxz;
  A[2][0] = Szx - Sxz; A[2][1] = Sxy + Syx; A[2][2] = -Sxx + Syy - Szz; A[2][3] = Syz + Szy;
  A[3][0] = Sxy - Syx; A[3][1] = Szx + Sxz; A[3][2] = Syz + Szy; A[3][3] = -Sxx - Syy + Szz;
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) V[r][c] = r == c ? 1.0 : 0.0;
  for (int sweep = 0; sweep < kJacobiSweeps; ++sweep) {
    const double off = A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[0][3] * A[0][3] +
                       A[1][2] * A[1][2] + A[1][3] * A[1][3] + A[2][3] * A[2][3];
    if (off < 1e-36) break;  // |entries| <= ~3 after normalisation: converged to fp64 round-off
    jacobi_rotate<0, 1>(A, V); jacobi_rotate<0, 2>(A, V); jacobi_rotate<0, 3>(A, V);
    jacobi_rotate<1, 2>(A, V); jacobi_rotate<1, 3>(A, V); jacobi_rotate<2, 3>(A, V);
  }
}

// Row-major rotation of the unit quaternion (w, x, y, z), applied as Q y to column vectors.
__device__ __forceinline__ void quat_rotation(double w, double x, double y, double z, double (&Q)[3][3]) {
  Q[0][0] = w * w + x * x - y * y - z * z; Q[0][1] = 2.0 * (x * y - w * z); Q[0][2] = 2.0 * (x * z + w * y);
  Q[1][0] = 2.0 * (x * y + w * z); Q[1][1] = w * w - x * x + y * y - z * z; Q[1][2] = 2.0 * (y * z - w * x);
  Q[2][0] = 2.0 * (x * z - w * y); Q[2][1] = 2.0 * (y * z + w * x); Q[2][2] = w * w - x * x - y * y + z * z;
}

}  // namespace
}  // namespace vp3d
