// sgr_meshbind.cu -- Gaussians bound to a triangle mesh (the refinement stage's per-step prologue).
//
// Replaces the PyTorch property code of a mesh-bound SuGaR model (reference: sugar_scene/sugar_model.py)
//   points       :384-398   barycentric combination of each face's vertices, n Gaussians per face
//   scaling      :415-441   (thickness, exp(_scales[:,0]), exp(_scales[:,1]))
//   quaternions  :443-479   frame (face normal | first edge rotated by the learned complex number | their
//                            cross product) -> matrix_to_quaternion -> normalize
// and its autograd: ~40 elementwise / gather / cross / normalize kernels with [F,n,3,3] temporaries per
// step.  One thread per FACE: the frame is built once and shared by the face's n Gaussians; in the backward
// the face's Gaussians are folded into the frame's adjoint first, so a face issues 9 atomics to its three
// vertices instead of 9 per Gaussian.
// The edited model (make_editable, get_edited_quaternions_and_scales :562-667) is a forward-only kernel of its own on
// the same frame: render-time arithmetic for a deformed or animated mesh.
//
// Third-party arithmetic restated from pytorch3d 0.7.4 (not under /root/reference):
//   Meshes.faces_normals_packed : n = (v1 - v0) x (v2 - v0), n / max(|n|, 1e-6)
//   matrix_to_quaternion        : the four candidates q_abs = sqrt(max(0, 1 +- m00 +- m11 +- m22)), the
//                                 row of the largest q_abs divided by 2 max(q_abs, 0.1)
#include <math.h>

#include "sgr_internal.cuh"

// The per-face arithmetic is plain C++: tests/test_meshbind_oracle.py compiles this file with
// -DSGR_MESHBIND_HOST_TEST and runs the same functions on the host against the oracle, so the hand-written
// adjoint is checked where there is no GPU.  The product library only contains the kernels.
#define SGR_HD __host__ __device__ __forceinline__

namespace sgr {

struct V3 {
    float x, y, z;
};
SGR_HD V3 operator+(V3 a, V3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
SGR_HD V3 operator-(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
SGR_HD V3 operator*(float s, V3 a) { return {s * a.x, s * a.y, s * a.z}; }
SGR_HD float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
SGR_HD V3 cross(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
SGR_HD V3 ld3(const float *p) { return {p[0], p[1], p[2]}; }

// y = x / max(|x|, eps)  and its adjoint  g_x = (g_y - y <y, g_y>) / |x|   (|x| > eps), g_y / eps otherwise
SGR_HD V3 normalize_eps(V3 x, float eps, float &len)
{
    len = sqrtf(dot(x, x));
    return (1.0f / fmaxf(len, eps)) * x;
}
SGR_HD V3 normalize_adj(V3 y, V3 gy, float len, float eps)
{
    if (len > eps) return (1.0f / len) * (gy - dot(y, gy) * y);
    return (1.0f / eps) * gy;
}

struct Frame {
    V3 v0, v1, v2;
    V3 a, b, nraw, fn, R0, e, R1b, c, R2b;
    float nlen, fnlen, elen, clen;
};

SGR_HD Frame face_frame(const float *__restrict__ verts, const int64_t *__restrict__ faces, int f)
{
    Frame F;
    F.v0 = ld3(verts + 3 * faces[3 * (size_t)f]);
    F.v1 = ld3(verts + 3 * faces[3 * (size_t)f + 1]);
    F.v2 = ld3(verts + 3 * faces[3 * (size_t)f + 2]);
    F.a = F.v1 - F.v0;
    F.b = F.v2 - F.v0;
    F.nraw = cross(F.a, F.b);
    F.fn = normalize_eps(F.nraw, 1e-6f, F.nlen);     // pytorch3d face normal
    F.R0 = normalize_eps(F.fn, 1e-12f, F.fnlen);     // sugar_model.py:448
    F.e = F.v0 - F.v1;                               // :452 "first side of every triangle"
    F.R1b = normalize_eps(F.e, 1e-12f, F.elen);
    F.c = cross(F.R0, F.R1b);                        // :455
    F.R2b = normalize_eps(F.c, 1e-12f, F.clen);
    return F;
}

// matrix_to_quaternion for R = [c0 | c1 | c2] (columns): returns the un-normalised candidate row, which
// branch k was taken, s = q_abs_k
SGR_HD void mat2quat(V3 c0, V3 c1, V3 c2, float q[4], int &k, float &s)
{
    const float m00 = c0.x, m10 = c0.y, m20 = c0.z, m01 = c1.x, m11 = c1.y, m21 = c1.z, m02 = c2.x, m12 = c2.y, m22 = c2.z;
    const float t[4] = {1.f + m00 + m11 + m22, 1.f + m00 - m11 - m22, 1.f - m00 + m11 - m22, 1.f - m00 - m11 + m22};
    float qa[4];
#pragma unroll
    for (int i = 0; i < 4; i++) qa[i] = t[i] > 0.f ? sqrtf(t[i]) : 0.f;
    k = 0;
#pragma unroll
    for (int i = 1; i < 4; i++)
        if (qa[i] > qa[k]) k = i;  // torch.argmax: first maximum
    s = qa[k];
    const float d = 1.0f / (2.0f * fmaxf(s, 0.1f));
    float N[4];
    if (k == 0) {
        N[0] = s * s; N[1] = m21 - m12; N[2] = m02 - m20; N[3] = m10 - m01;
    } else if (k == 1) {
        N[0] = m21 - m12; N[1] = s * s; N[2] = m10 + m01; N[3] = m02 + m20;
    } else if (k == 2) {
        N[0] = m02 - m20; N[1] = m10 + m01; N[2] = s * s; N[3] = m12 + m21;
    } else {
        N[0] = m10 - m01; N[1] = m20 + m02; N[2] = m21 + m12; N[3] = s * s;
    }
#pragma unroll
    for (int i = 0; i < 4; i++) q[i] = N[i] * d;
}

// adjoint of mat2quat: g_q (wrt the un-normalised candidate) -> g_c0, g_c1, g_c2
SGR_HD void mat2quat_adj(V3 c0, V3 c1, V3 c2, const float q[4], int k, float s, const float gq[4], V3 &g0,
                                             V3 &g1, V3 &g2)
{
    const float dd = 2.0f * fmaxf(s, 0.1f), d = 1.0f / dd;
    float gN[4], gd = 0.f;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        gN[i] = gq[i] * d;
        gd -= gq[i] * q[i] * d;  // q = N / dd  ->  dq/ddd = -q / dd
    }
    float gs = 2.0f * s * gN[k];      // N_k = s^2
    if (s > 0.1f) gs += 2.0f * gd;    // dd = 2 s
    const float gt = s > 0.f ? gs / (2.0f * s) : 0.f;  // s = sqrt(t), zero subgradient at t <= 0
    // t_k = 1 + sg0 m00 + sg1 m11 + sg2 m22
    const float sg0 = (k == 0 || k == 1) ? 1.f : -1.f, sg1 = (k == 0 || k == 2) ? 1.f : -1.f, sg2 = (k == 0 || k == 3) ? 1.f : -1.f;
    float g00 = sg0 * gt, g11 = sg1 * gt, g22 = sg2 * gt;
    float g01 = 0.f, g02 = 0.f, g10 = 0.f, g12 = 0.f, g20 = 0.f, g21 = 0.f;
    if (k == 0) {
        g21 += gN[1]; g12 -= gN[1]; g02 += gN[2]; g20 -= gN[2]; g10 += gN[3]; g01 -= gN[3];
    } else if (k == 1) {
        g21 += gN[0]; g12 -= gN[0]; g10 += gN[2]; g01 += gN[2]; g02 += gN[3]; g20 += gN[3];
    } else if (k == 2) {
        g02 += gN[0]; g20 -= gN[0]; g10 += gN[1]; g01 += gN[1]; g12 += gN[3]; g21 += gN[3];
    } else {
        g10 += gN[0]; g01 -= gN[0]; g20 += gN[1]; g02 += gN[1]; g21 += gN[2]; g12 += gN[2];
    }
    // m_ij = (column j)_i
    g0 = {g00, g10, g20};
    g1 = {g01, g11, g21};
    g2 = {g02, g12, g22};
}

SGR_HD void meshbind_face_forward(int f, int n_per, const float *__restrict__ verts, const int64_t *__restrict__ faces,
                                  const float *__restrict__ bary, const float *__restrict__ scales_raw,
                                  const float *__restrict__ complex_raw, float thickness, float *__restrict__ points,
                                  float *__restrict__ scaling, float *__restrict__ quats)
{
    const Frame fr = face_frame(verts, faces, f);
    for (int n = 0; n < n_per; n++) {
        const size_t g = (size_t)f * n_per + n;
        const float b0 = bary[3 * n], b1 = bary[3 * n + 1], b2 = bary[3 * n + 2];
        const V3 p = (b0 * fr.v0 + b1 * fr.v1) + b2 * fr.v2;
        points[3 * g] = p.x;
        points[3 * g + 1] = p.y;
        points[3 * g + 2] = p.z;
        scaling[3 * g] = thickness;
        scaling[3 * g + 1] = expf(scales_raw[2 * g]);
        scaling[3 * g + 2] = expf(scales_raw[2 * g + 1]);
        const float cr = complex_raw[2 * g], ci = complex_raw[2 * g + 1];
        const float cl = 1.0f / fmaxf(sqrtf(cr * cr + ci * ci), 1e-12f);
        const float zr = cr * cl, zi = ci * cl;
        const V3 R1 = zr * fr.R1b + zi * fr.R2b, R2 = (-zi) * fr.R1b + zr * fr.R2b;
        float q[4], s;
        int k;
        mat2quat(fr.R0, R1, R2, q, k, s);
        const float ql = 1.0f / fmaxf(sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]), 1e-12f);
        quats[4 * g] = q[0] * ql;
        quats[4 * g + 1] = q[1] * ql;
        quats[4 * g + 2] = q[2] * ql;
        quats[4 * g + 3] = q[3] * ql;
    }
}

// y = x / max(|x|, eps), divided as F.normalize divides (the edited binding's vertex axes)
SGR_HD V3 normalize_div(V3 x, float eps, float &len)
{
    len = sqrtf(dot(x, x));
    const float d = fmaxf(len, eps);
    return {x.x / d, x.y / d, x.z / d};
}

// The face's vertex axes normalize(mean - v_k) and their lengths (sugar_model.py:636-642).  The angle axes of :598-603,
// normalize(v_k - mean) with the third one negated, are (-A_0, -A_1, A_2) exactly: negation commutes with every rounding.
SGR_HD void vertex_axes(V3 v0, V3 v1, V3 v2, V3 A[3], float len[3])
{
    const V3 s = (v0 + v1) + v2, m = {s.x / 3.0f, s.y / 3.0f, s.z / 3.0f};
    A[0] = normalize_div(m - v0, 1e-12f, len[0]);
    A[1] = normalize_div(m - v1, 1e-12f, len[1]);
    A[2] = normalize_div(m - v2, 1e-12f, len[2]);
}

// arccos(clamp(<angle axis k, base>, -1, 1)) for the three axes (:606-607)
SGR_HD void axis_angles(const V3 A[3], V3 base, float ang[3])
{
    const float sg[3] = {-1.f, -1.f, 1.f};
#pragma unroll
    for (int k = 0; k < 3; k++) ang[k] = acosf(fminf(fmaxf(sg[k] * dot(A[k], base), -1.f), 1.f));
}

// The edited model's Gaussians of face f (get_edited_quaternions_and_scales, sugar_model.py:572-667, with the
// `quaternions` / `scaling` properties' final normalize and plane-scale product): the face frame of bind_to_mesh at the
// current vertices, each Gaussian's learned in-plane rotation turned by the bary-weighted change of the vertex-axis
// angles, and each plane scale stretched by the bary-weighted change of the axis lengths, both against the reference
// vertices.  Gaussian g is written to row out_rows[g] (skipped when negative), or to row g - row0 when out_rows is NULL.
SGR_HD void meshbind_face_edited_forward(int f, int n_per, const float *__restrict__ verts,
                                         const float *__restrict__ reference_verts, const int64_t *__restrict__ faces,
                                         const float *__restrict__ bary, const float *__restrict__ scales_raw,
                                         const float *__restrict__ complex_raw, float thickness,
                                         const int64_t *__restrict__ out_rows, int64_t row0, float *__restrict__ points,
                                         float *__restrict__ scaling, float *__restrict__ quats)
{
    const Frame fr = face_frame(verts, faces, f);
    const V3 r0 = ld3(reference_verts + 3 * faces[3 * (size_t)f]), r1 = ld3(reference_verts + 3 * faces[3 * (size_t)f + 1]),
             r2 = ld3(reference_verts + 3 * faces[3 * (size_t)f + 2]);
    V3 A[3], RA[3];
    float len[3], rlen[3], ang[3], rang[3], blen;
    vertex_axes(fr.v0, fr.v1, fr.v2, A, len);
    vertex_axes(r0, r1, r2, RA, rlen);
    axis_angles(A, fr.R1b, ang);                                   // faces_base is bind_to_mesh's base_R_1
    axis_angles(RA, normalize_eps(r0 - r1, 1e-12f, blen), rang);   // the same normalize: equal vertices, equal angles
    float dang[3];
    V3 O[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        dang[k] = ang[k] - rang[k];
        O[k] = cross(A[k], fr.fn);                                 // :639, against the pytorch3d face normal
    }
    for (int n = 0; n < n_per; n++) {
        const size_t g = (size_t)f * n_per + n;
        const int64_t row = out_rows ? out_rows[g] : (int64_t)g - row0;
        if (row < 0) continue;
        const float b0 = bary[3 * n], b1 = bary[3 * n + 1], b2 = bary[3 * n + 2];
        const V3 p = (b0 * fr.v0 + b1 * fr.v1) + b2 * fr.v2;
        points[3 * row] = p.x;
        points[3 * row + 1] = p.y;
        points[3 * row + 2] = p.z;
        // the learned complex number turned by the point's angle (:608-621)
        const float pa = (dang[0] * b0 + dang[1] * b1) + dang[2] * b2;
        float sa, ca;
        sincosf(pa, &sa, &ca);
        const float cr = complex_raw[2 * g], ci = complex_raw[2 * g + 1];
        const float cl = 1.0f / fmaxf(sqrtf(cr * cr + ci * ci), 1e-12f);
        const float x = cr * cl, y = ci * cl;
        const float zr = x * ca - y * sa, zi = x * sa + y * ca;
        const V3 R1 = zr * fr.R1b + zi * fr.R2b, R2 = (-zi) * fr.R1b + zr * fr.R2b;
        float q[4], s;
        int k;
        mat2quat(fr.R0, R1, R2, q, k, s);
        const float ql = 1.0f / fmaxf(sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]), 1e-12f);
        quats[4 * row] = q[0] * ql;
        quats[4 * row + 1] = q[1] * ql;
        quats[4 * row + 2] = q[2] * ql;
        quats[4 * row + 3] = q[3] * ql;
        // stretch of each in-plane axis along the vertex axes (:644-660)
        float st1[3], st2[3];
#pragma unroll
        for (int j = 0; j < 3; j++) {
            const float a1 = dot(R1, A[j]) * len[j] / rlen[j], o1 = dot(R1, O[j]);
            const float a2 = dot(R2, A[j]) * len[j] / rlen[j], o2 = dot(R2, O[j]);
            st1[j] = sqrtf(a1 * a1 + o1 * o1);
            st2[j] = sqrtf(a2 * a2 + o2 * o2);
        }
        scaling[3 * row] = thickness;
        scaling[3 * row + 1] = expf(scales_raw[2 * g]) * ((st1[0] * b0 + st1[1] * b1) + st1[2] * b2);
        scaling[3 * row + 2] = expf(scales_raw[2 * g + 1]) * ((st2[0] * b0 + st2[1] * b1) + st2[2] * b2);
    }
}

SGR_HD void vadd(float *p, float v)
{
#ifdef __CUDA_ARCH__
    atomicAdd(p, v);
#else
    *p += v;
#endif
}

SGR_HD void meshbind_face_backward(int f, int n_per, const float *__restrict__ verts, const int64_t *__restrict__ faces,
                                   const float *__restrict__ bary, const float *__restrict__ scales_raw,
                                   const float *__restrict__ complex_raw, const float *__restrict__ g_points,
                                   const float *__restrict__ g_scaling, const float *__restrict__ g_quats,
                                   float *__restrict__ g_verts, float *__restrict__ g_scales_raw,
                                   float *__restrict__ g_complex_raw)
{
    const Frame fr = face_frame(verts, faces, f);
    V3 gv0 = {0, 0, 0}, gv1 = {0, 0, 0}, gv2 = {0, 0, 0};
    V3 gR0 = {0, 0, 0}, gR1b = {0, 0, 0}, gR2b = {0, 0, 0};
    for (int n = 0; n < n_per; n++) {
        const size_t g = (size_t)f * n_per + n;
        // points
        const V3 gp = ld3(g_points + 3 * g);
        gv0 = gv0 + bary[3 * n] * gp;
        gv1 = gv1 + bary[3 * n + 1] * gp;
        gv2 = gv2 + bary[3 * n + 2] * gp;
        // scaling: d exp
        g_scales_raw[2 * g] = g_scaling[3 * g + 1] * expf(scales_raw[2 * g]);
        g_scales_raw[2 * g + 1] = g_scaling[3 * g + 2] * expf(scales_raw[2 * g + 1]);
        // quaternion: recompute the forward chain of this Gaussian, then walk it backwards
        const float cr = complex_raw[2 * g], ci = complex_raw[2 * g + 1];
        const float clen = sqrtf(cr * cr + ci * ci), cl = 1.0f / fmaxf(clen, 1e-12f);
        const float zr = cr * cl, zi = ci * cl;
        const V3 R1 = zr * fr.R1b + zi * fr.R2b, R2 = (-zi) * fr.R1b + zr * fr.R2b;
        float q[4], s;
        int k;
        mat2quat(fr.R0, R1, R2, q, k, s);
        const float qlen = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]), ql = 1.0f / fmaxf(qlen, 1e-12f);
        float gqn[4] = {g_quats[4 * g], g_quats[4 * g + 1], g_quats[4 * g + 2], g_quats[4 * g + 3]}, gq[4];
        if (qlen > 1e-12f) {
            const float qd = (q[0] * gqn[0] + q[1] * gqn[1] + q[2] * gqn[2] + q[3] * gqn[3]) * ql * ql;  // <qn, g> / |q|
#pragma unroll
            for (int i = 0; i < 4; i++) gq[i] = gqn[i] * ql - q[i] * qd * ql;
        } else {
#pragma unroll
            for (int i = 0; i < 4; i++) gq[i] = gqn[i] * 1e12f;
        }
        V3 g0, g1, g2;
        mat2quat_adj(fr.R0, R1, R2, q, k, s, gq, g0, g1, g2);
        gR0 = gR0 + g0;
        // R1 = zr R1b + zi R2b, R2 = -zi R1b + zr R2b
        const float gzr = dot(g1, fr.R1b) + dot(g2, fr.R2b), gzi = dot(g1, fr.R2b) - dot(g2, fr.R1b);
        gR1b = gR1b + (zr * g1 - zi * g2);
        gR2b = gR2b + (zi * g1 + zr * g2);
        // z = c / |c|
        if (clen > 1e-12f) {
            const float zd = zr * gzr + zi * gzi;
            g_complex_raw[2 * g] = (gzr - zr * zd) * cl;
            g_complex_raw[2 * g + 1] = (gzi - zi * zd) * cl;
        } else {
            g_complex_raw[2 * g] = gzr * 1e12f;
            g_complex_raw[2 * g + 1] = gzi * 1e12f;
        }
    }
    // frame adjoint: R2b = normalize(R0 x R1b), R1b = normalize(v0 - v1), R0 = normalize(normalize_1e-6((v1-v0) x (v2-v0)))
    const V3 gc = normalize_adj(fr.R2b, gR2b, fr.clen, 1e-12f);
    gR0 = gR0 + cross(fr.R1b, gc);
    gR1b = gR1b + cross(gc, fr.R0);
    const V3 ge = normalize_adj(fr.R1b, gR1b, fr.elen, 1e-12f);
    gv0 = gv0 + ge;
    gv1 = gv1 - ge;
    const V3 gfn = normalize_adj(fr.R0, gR0, fr.fnlen, 1e-12f);
    const V3 gn = normalize_adj(fr.fn, gfn, fr.nlen, 1e-6f);
    const V3 ga = cross(fr.b, gn), gb = cross(gn, fr.a);
    gv1 = gv1 + ga;
    gv2 = gv2 + gb;
    gv0 = gv0 - (ga + gb);
    float *o0 = g_verts + 3 * faces[3 * (size_t)f], *o1 = g_verts + 3 * faces[3 * (size_t)f + 1],
          *o2 = g_verts + 3 * faces[3 * (size_t)f + 2];
    vadd(o0, gv0.x); vadd(o0 + 1, gv0.y); vadd(o0 + 2, gv0.z);
    vadd(o1, gv1.x); vadd(o1 + 1, gv1.y); vadd(o1 + 2, gv1.z);
    vadd(o2, gv2.x); vadd(o2 + 1, gv2.y); vadd(o2 + 2, gv2.z);
}

__global__ void __launch_bounds__(128) meshbind_forward_kernel(int F, int n_per, const float *__restrict__ verts,
                                                               const int64_t *__restrict__ faces,
                                                               const float *__restrict__ bary,
                                                               const float *__restrict__ scales_raw,
                                                               const float *__restrict__ complex_raw, float thickness,
                                                               float *__restrict__ points, float *__restrict__ scaling,
                                                               float *__restrict__ quats)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f < F) meshbind_face_forward(f, n_per, verts, faces, bary, scales_raw, complex_raw, thickness, points, scaling, quats);
}

// Without out_rows a CTA's Gaussians are one contiguous run of rows: they are staged in shared memory (10 floats each)
// and leave in coalesced stores.  Stored straight from each thread, n_per > 1 rows per thread put every store
// instruction on 32 separate sectors (4x slower at n_per = 6, measured).  out_rows scatters anyway and stores directly.
constexpr int EDIT_T = 128;
constexpr int EDIT_STAGE_MAX_N = 9;   // 128 faces x 9 Gaussians x 40 B = 45 KB of shared memory

__global__ void __launch_bounds__(EDIT_T) meshbind_edited_forward_kernel(
    int F, int n_per, const float *__restrict__ verts, const float *__restrict__ reference_verts,
    const int64_t *__restrict__ faces, const float *__restrict__ bary, const float *__restrict__ scales_raw,
    const float *__restrict__ complex_raw, float thickness, const int64_t *__restrict__ out_rows, int staged,
    float *__restrict__ points, float *__restrict__ scaling, float *__restrict__ quats)
{
    const int f = blockIdx.x * EDIT_T + threadIdx.x;
    if (!staged) {
        if (f < F)
            meshbind_face_edited_forward(f, n_per, verts, reference_verts, faces, bary, scales_raw, complex_raw,
                                         thickness, out_rows, 0, points, scaling, quats);
        return;
    }
    extern __shared__ float s_rows[];
    float *sp = s_rows, *ss = sp + 3 * EDIT_T * n_per, *sq = ss + 3 * EDIT_T * n_per;
    const int64_t g0 = (int64_t)blockIdx.x * EDIT_T * n_per;
    const int cnt = min(EDIT_T, F - (int)(blockIdx.x * EDIT_T)) * n_per;
    if (f < F)
        meshbind_face_edited_forward(f, n_per, verts, reference_verts, faces, bary, scales_raw, complex_raw, thickness,
                                     nullptr, g0, sp, ss, sq);
    __syncthreads();
    for (int i = threadIdx.x; i < 3 * cnt; i += EDIT_T) {
        points[3 * g0 + i] = sp[i];
        scaling[3 * g0 + i] = ss[i];
    }
    for (int i = threadIdx.x; i < 4 * cnt; i += EDIT_T) quats[4 * g0 + i] = sq[i];
}

__global__ void __launch_bounds__(128) meshbind_backward_kernel(int F, int n_per, const float *__restrict__ verts,
                                                                const int64_t *__restrict__ faces,
                                                                const float *__restrict__ bary,
                                                                const float *__restrict__ scales_raw,
                                                                const float *__restrict__ complex_raw,
                                                                const float *__restrict__ g_points,
                                                                const float *__restrict__ g_scaling,
                                                                const float *__restrict__ g_quats, float *__restrict__ g_verts,
                                                                float *__restrict__ g_scales_raw,
                                                                float *__restrict__ g_complex_raw)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f < F)
        meshbind_face_backward(f, n_per, verts, faces, bary, scales_raw, complex_raw, g_points, g_scaling, g_quats, g_verts,
                               g_scales_raw, g_complex_raw);
}

}  // namespace sgr

using namespace sgr;

#ifdef SGR_MESHBIND_HOST_TEST
// test-only build (never part of libsugar_b200.so): the same per-face functions, looped on the host
extern "C" void meshbind_host_forward(int F, int n_per, const float *verts, const int64_t *faces, const float *bary,
                                      const float *scales_raw, const float *complex_raw, float thickness, float *points,
                                      float *scaling, float *quats)
{
    for (int f = 0; f < F; f++)
        meshbind_face_forward(f, n_per, verts, faces, bary, scales_raw, complex_raw, thickness, points, scaling, quats);
}
extern "C" void meshbind_host_backward(int F, int n_per, const float *verts, const int64_t *faces, const float *bary,
                                       const float *scales_raw, const float *complex_raw, const float *g_points,
                                       const float *g_scaling, const float *g_quats, float *g_verts, float *g_scales_raw,
                                       float *g_complex_raw)
{
    for (int f = 0; f < F; f++)
        meshbind_face_backward(f, n_per, verts, faces, bary, scales_raw, complex_raw, g_points, g_scaling, g_quats, g_verts,
                               g_scales_raw, g_complex_raw);
}
extern "C" void meshbind_host_edited_forward(int F, int n_per, const float *verts, const float *reference_verts,
                                             const int64_t *faces, const float *bary, const float *scales_raw,
                                             const float *complex_raw, float thickness, const int64_t *out_rows,
                                             float *points, float *scaling, float *quats)
{
    for (int f = 0; f < F; f++)
        meshbind_face_edited_forward(f, n_per, verts, reference_verts, faces, bary, scales_raw, complex_raw, thickness,
                                     out_rows, 0, points, scaling, quats);
}
#else
extern "C" int sgr_meshbind_forward(int32_t F, int32_t n_per, int32_t V, const float *verts, const int64_t *faces,
                                    const float *bary, const float *scales_raw, const float *complex_raw, float thickness,
                                    float *points, float *scaling, float *quaternions, void *stream)
{
    if (F < 0 || n_per <= 0 || V < 0 ||
        (F > 0 && (!verts || !faces || !bary || !scales_raw || !complex_raw || !points || !scaling || !quaternions))) {
        set_error("bad arguments to sgr_meshbind_forward");
        return SGR_EINVAL;
    }
    if (F == 0) return SGR_OK;
    cudaStream_t st = (cudaStream_t)stream;
    SGR_LAUNCH(K_MISC, st,
               meshbind_forward_kernel<<<(F + 127) / 128, 128, 0, st>>>(F, n_per, verts, faces, bary, scales_raw, complex_raw,
                                                                       thickness, points, scaling, quaternions));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

extern "C" int sgr_meshbind_edited_forward(int32_t F, int32_t n_per, int32_t V, const float *verts,
                                           const float *reference_verts, const int64_t *faces, const float *bary,
                                           const float *scales_raw, const float *complex_raw, float thickness,
                                           const int64_t *out_rows, float *points, float *scaling, float *quaternions,
                                           void *stream)
{
    if (F < 0 || n_per <= 0 || V < 0 ||
        (F > 0 && (!verts || !reference_verts || !faces || !bary || !scales_raw || !complex_raw || !points || !scaling ||
                   !quaternions))) {
        set_error("bad arguments to sgr_meshbind_edited_forward");
        return SGR_EINVAL;
    }
    if (F == 0) return SGR_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const int staged = !out_rows && n_per <= EDIT_STAGE_MAX_N;
    const size_t smem = staged ? sizeof(float) * 10 * EDIT_T * n_per : 0;
    SGR_LAUNCH(K_MISC, st,
               meshbind_edited_forward_kernel<<<(F + EDIT_T - 1) / EDIT_T, EDIT_T, smem, st>>>(
                   F, n_per, verts, reference_verts, faces, bary, scales_raw, complex_raw, thickness, out_rows, staged,
                   points, scaling, quaternions));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

extern "C" int sgr_meshbind_backward(int32_t F, int32_t n_per, int32_t V, const float *verts, const int64_t *faces,
                                     const float *bary, const float *scales_raw, const float *complex_raw,
                                     const float *g_points, const float *g_scaling, const float *g_quaternions,
                                     float *g_verts, float *g_scales_raw, float *g_complex_raw, void *stream)
{
    if (F < 0 || n_per <= 0 || V < 0 ||
        (F > 0 && (!verts || !faces || !bary || !scales_raw || !complex_raw || !g_points || !g_scaling ||
                   !g_quaternions || !g_verts || !g_scales_raw || !g_complex_raw))) {
        set_error("bad arguments to sgr_meshbind_backward");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (V > 0) SGR_CUDA(cudaMemsetAsync(g_verts, 0, sizeof(float) * 3 * (size_t)V, st));
    if (F == 0) return SGR_OK;
    SGR_LAUNCH(K_MISC, st,
               meshbind_backward_kernel<<<(F + 127) / 128, 128, 0, st>>>(F, n_per, verts, faces, bary, scales_raw,
                                                                        complex_raw, g_points, g_scaling, g_quaternions,
                                                                        g_verts, g_scales_raw, g_complex_raw));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}
#endif  // SGR_MESHBIND_HOST_TEST
