// The camera projection of common/camera.py:37-88 for one point, in fp32, and its reverse mode:
// perspective divide clamped to [-1, 1], radial k1..k3 and tangential p1, p2 distortion, focal
// length and principal point (:37-67), or only the linear part (:69-88).  Shared by the
// re-projection loss (step_ops.cu) and the unlabeled pass of the semi-supervised head (semi_loss.cu),
// which must give the same bits for the same point.
#pragma once

namespace vp3d {
namespace {

struct Camera {  // the 9 intrinsics in camera.py's order
  float fx, fy, cx, cy, k0, k1, k2, p0, p1;
};

__device__ __forceinline__ Camera load_camera(const float* c) {
  return {c[0], c[1], c[2], c[3], c[4], c[5], c[6], c[7], c[8]};
}

struct Projection {
  float x, y;    // the projected point
  float u, v;    // perspective divide, before the clamp
  float xx, yy;  // u, v clamped to [-1, 1]
  float z;       // depth
  float s, rp;   // distortion factor and d radial / d r2 (1 and 0 in the linear form)
};

__device__ __forceinline__ Projection project(const Camera& c, float x, float y, float z, bool linear) {
  Projection P;
  P.u = x / z; P.v = y / z; P.z = z;
  P.xx = fminf(fmaxf(P.u, -1.0f), 1.0f); P.yy = fminf(fmaxf(P.v, -1.0f), 1.0f);
  float ox, oy;  // projected point before focal length / principal point
  P.s = 1.0f; P.rp = 0.0f;
  if (linear) {
    ox = P.xx; oy = P.yy;
  } else {
    const float r2 = P.xx * P.xx + P.yy * P.yy;
    const float radial = 1.0f + r2 * (c.k0 + r2 * (c.k1 + r2 * c.k2));
    P.rp = c.k0 + r2 * (2.0f * c.k1 + 3.0f * c.k2 * r2);
    P.s = radial + (c.p0 * P.xx + c.p1 * P.yy);
    ox = P.xx * P.s + c.p0 * r2;
    oy = P.yy * P.s + c.p1 * r2;
  }
  P.x = c.fx * ox + c.cx; P.y = c.fy * oy + c.cy;
  return P;
}

// d loss / d (x, y, z) of the point given d loss / d (P.x, P.y) = (ex, ey) * inv.  The scale inv is
// a separate argument because the focal length multiplies (ex, ey) before it does.
__device__ __forceinline__ float3 project_backward(const Camera& c, const Projection& P, float ex, float ey,
                                                   float inv, bool linear) {
  const float a = c.fx * ex * inv, b = c.fy * ey * inv;  // d loss / d (ox, oy)
  float gxx, gyy;
  if (linear) {
    gxx = a; gyy = b;
  } else {
    const float sx = P.rp * 2.0f * P.xx + c.p0, sy = P.rp * 2.0f * P.yy + c.p1;  // d s / d (xx, yy)
    gxx = a * (P.s + P.xx * sx + c.p0 * 2.0f * P.xx) + b * (P.yy * sx + c.p1 * 2.0f * P.xx);
    gyy = a * (P.xx * sy + c.p0 * 2.0f * P.yy) + b * (P.s + P.yy * sy + c.p1 * 2.0f * P.yy);
  }
  const float gu = (P.u >= -1.0f && P.u <= 1.0f) ? gxx : 0.0f;  // clamp passes gradient inside
  const float gv = (P.v >= -1.0f && P.v <= 1.0f) ? gyy : 0.0f;
  return make_float3(gu / P.z, gv / P.z, -(gu * P.u + gv * P.v) / P.z);
}

}  // namespace
}  // namespace vp3d
