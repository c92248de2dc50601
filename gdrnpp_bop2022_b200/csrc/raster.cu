// CUDA depth rasteriser (no EGL / GL interop) + the fast depth-refinement step.
//
// Replaces, for depth output, lib/render_vispy/renderer.py:126-182,363-407,461-476 (the renderer
// fast depth refine calls) and lib/egl_renderer/egl_renderer_v3.py:755-783,838-1228 (pc_cam[...,2]).
// GL conventions reproduced (SURVEY.md Appendix B): camera-space (X,Y,Z) in OpenCV axes projects to
// u = fx*X/Z + skew*Y/Z + cx, v = fy*Y/Z + cy; pixel (row r, col c) is sampled at (c+0.5, r+0.5);
// coverage = sample inside the projected triangle (either winding, no culling: renderer.py:102);
// the z-buffer value is affine in window space, i.e. 1/Z is interpolated with screen-space
// barycentrics (== the perspective-correct interpolation of camera-space Z in the EGL shader);
// nearest fragment wins, and on equal depth the lower triangle index; background = 0.  Triangles with a vertex closer
// than znear are dropped whole (GL would clip them; objects in front of the camera never hit this); a fragment with
// z < znear or z > zfar is dropped at its pixel.  Coverage is watertight: the triangles sharing an edge evaluate its
// edge function bit for bit alike up to sign (edge_fn), so a sample on the shared side of one is covered by the other.
//
// Algorithmic HBM traffic per render: 12*V + 12*F bytes of mesh + 8*H*W z-buffer scratch + 4*H*W out.
// One thread per (render, triangle); 64-bit atomicMin on (z_bits << 32 | triangle) resolves visibility.
#include "common.cuh"

namespace {

// Edge function of the edge a -> b at the sample (sx, sy), (ua - sx)(vb - sy) - (ub - sx)(va - sy).  The endpoints are
// taken in a canonical order (by screen position) and the products are not contracted into an fma, so the two
// triangles sharing an edge get the same magnitude with opposite signs whatever their vertex order: a sample is covered
// by at least one of them, and by both only when it lies exactly on the edge.
__device__ __forceinline__ float edge_fn(float ua, float va, float ub, float vb, float sx, float sy) {
  const bool swap = ub < ua || (ub == ua && vb < va);
  const float x0 = swap ? ub : ua, y0 = swap ? vb : va, x1 = swap ? ua : ub, y1 = swap ? va : vb;
  const float e = __fsub_rn(__fmul_rn(__fsub_rn(x0, sx), __fsub_rn(y1, sy)), __fmul_rn(__fsub_rn(x1, sx), __fsub_rn(y0, sy)));
  return swap ? -e : e;
}

__global__ void rast_clear_kernel(unsigned long long* zbuf, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    zbuf[i] = 0xFFFFFFFFFFFFFFFFull;
}

// ---- mesh registry: meshes uploaded once (rast_upload_mesh), renders pick one per ROI by id --------------------------
struct MeshEntry {
  const float* verts;
  const int* faces;
  int V, F;
};
constexpr int RAST_MAX_MESHES = 1024;

// Per-mesh shading attributes of rast_upload_mesh_tex; null / 0 for what a mesh was uploaded without.
constexpr int RAST_MAX_MIPS = 16;
struct MeshTex {
  const float* normals;                    // [V,3] model-space vertex normals
  const float* uvs;                        // [V,2] per-vertex texture coordinates
  const uint8_t* tex;                      // mip chain: level l is [h[l], w[l], 3] u8 at tex + off[l], row 0 at t = 0
  int levels;                              // 0 = no texture
  int w[RAST_MAX_MIPS], h[RAST_MAX_MIPS];
  long long off[RAST_MAX_MIPS];
};

// the triangles of one ROI: mesh `mid` (an unknown id renders as background) at pose P [3,4] with intrinsics K, into zb.
// The key's low word is tri_base + the triangle's index in the mesh.
__device__ __forceinline__ void rast_tri_one(const MeshEntry* __restrict__ table, int mid, int n_meshes,
                                             const float* __restrict__ P, const float* __restrict__ K, int H, int W,
                                             float znear, float zfar, unsigned long long* __restrict__ zb,
                                             unsigned tri_base = 0u) {
  if (mid < 0 || mid >= n_meshes) return;
  const MeshEntry me = table[mid];
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= me.F) return;
  float u[3], v[3], iz[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int vi = me.faces[f * 3 + k];
    const float x = me.verts[vi * 3], y = me.verts[vi * 3 + 1], z = me.verts[vi * 3 + 2];
    const float X = P[0] * x + P[1] * y + P[2] * z + P[3];
    const float Y = P[4] * x + P[5] * y + P[6] * z + P[7];
    const float Z = P[8] * x + P[9] * y + P[10] * z + P[11];
    if (Z < znear) return;
    iz[k] = 1.0f / Z;
    u[k] = (K[0] * X + K[1] * Y) * iz[k] + K[2];
    v[k] = (K[4] * Y) * iz[k] + K[5];
  }
  const float area = (u[1] - u[0]) * (v[2] - v[0]) - (u[2] - u[0]) * (v[1] - v[0]);
  if (area == 0.f) return;
  const float inv_area = 1.0f / area;
  int c0 = max(0, (int)floorf(fminf(fminf(u[0], u[1]), u[2]) - 0.5f));
  int c1 = min(W - 1, (int)ceilf(fmaxf(fmaxf(u[0], u[1]), u[2]) - 0.5f));
  int r0 = max(0, (int)floorf(fminf(fminf(v[0], v[1]), v[2]) - 0.5f));
  int r1 = min(H - 1, (int)ceilf(fmaxf(fmaxf(v[0], v[1]), v[2]) - 0.5f));
  for (int py = r0; py <= r1; ++py) {
    const float sy = (float)py + 0.5f;
    for (int px = c0; px <= c1; ++px) {
      const float sx = (float)px + 0.5f;
      const float w0 = edge_fn(u[1], v[1], u[2], v[2], sx, sy) * inv_area;
      const float w1 = edge_fn(u[2], v[2], u[0], v[0], sx, sy) * inv_area;
      const float e2 = edge_fn(u[0], v[0], u[1], v[1], sx, sy) * inv_area;
      if (w0 < 0.f || w1 < 0.f || e2 < 0.f) continue;
      const float w2 = 1.0f - w0 - w1;   // interpolation weights that sum to 1: a plane of constant Z keeps its depth
      const float izp = w0 * iz[0] + w1 * iz[1] + w2 * iz[2];
      const float zp = 1.0f / izp;
      if (!(zp >= znear) || zp > zfar) continue;
      const unsigned long long key = ((unsigned long long)__float_as_uint(zp) << 32) | (tri_base + (unsigned)f);
      atomicMin(zb + (long long)py * W + px, key);
    }
  }
}

// one thread per (ROI, triangle of that ROI's mesh); grid.x covers the largest registered mesh, grid.y strides over
// the ROIs (gridDim.y is capped at 65535, so each block row may take several ROIs)
__global__ void __launch_bounds__(256)
rast_tri_multi_kernel(const MeshEntry* __restrict__ table, const int* __restrict__ mesh_ids, int n_meshes, int n,
                      const float* __restrict__ poses, const float* __restrict__ Ks, int H, int W, float znear, float zfar,
                      unsigned long long* __restrict__ zbuf) {
  for (int r = blockIdx.y; r < n; r += gridDim.y) rast_tri_one(table, mesh_ids[r], n_meshes, poses + r * 12, Ks + r * 9,
                                                               H, W, znear, zfar, zbuf + (long long)r * H * W);
}

__global__ void rast_resolve_kernel(const unsigned long long* __restrict__ zbuf, const float* __restrict__ Ks, int n,
                                    int H, int W, float znear, float zfar, int quantize_bits,
                                    float* __restrict__ depth, float* __restrict__ xyz_cam) {
  const long long total = (long long)n * H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long key = zbuf[i];
    float z = 0.f;
    if (key != 0xFFFFFFFFFFFFFFFFull) {
      z = __uint_as_float((unsigned)(key >> 32));
      if (quantize_bits > 0) {
        // fixed-point window depth d = (1/z - 1/n) / (1/f - 1/n), read back as float32 and decoded like
        // renderer.py:176-182: dep = mult / (d + addi)
        const double dn = (double)znear, df = (double)zfar;
        double d = (1.0 / (double)z - 1.0 / dn) / (1.0 / df - 1.0 / dn);
        const double q = (double)((1ull << quantize_bits) - 1);
        d = floor(d * q + 0.5) / q;
        const float dfl = (float)d;
        const float mult = (float)((dn * df) / (dn - df)), addi = (float)(df / (dn - df));
        z = (dfl == 1.0f) ? 0.f : mult / (dfl + addi);
      }
    }
    depth[i] = z;
    if (xyz_cam) {
      const int px = (int)(i % W), py = (int)((i / W) % H);
      const int r = (int)(i / ((long long)H * W));
      const float* K = Ks + r * 9;
      float X = 0.f, Y = 0.f;
      if (z > 0.f) {
        Y = ((float)py + 0.5f - K[5]) / K[4] * z;
        X = ((float)px + 0.5f - K[2] - K[1] * Y / z) / K[0] * z;
      }
      xyz_cam[i * 3] = X; xyz_cam[i * 3 + 1] = Y; xyz_cam[i * 3 + 2] = z;
    }
  }
}

// Colour resolve: each covered pixel's winning triangle (the low word of the rasteriser's key) is shaded with
// renderer_py's flat fragment shader (lib/pysixd/renderer_py.py:52-75), light at the eye origin, ambient 0.5:
//   L = normalize(interp(normalize(-P_k))),  n = face normal turned toward the viewer,
//   rgb = rint(min(0.5 + max(dot(L, n), 0), 1) * colour * 255).
// The screen barycentrics are recomputed with the rasteriser's arithmetic and made perspective-correct
// (b_k = w_k / Z_k / sum(w / Z)), which is how GL interpolates v_L and v_color.  The face normal of a plane through
// the eye-facing side satisfies dot(n, P) <= 0 for every point P of the triangle, so it is turned once per triangle.
// Colour: colors [n,3] per render when given, else the mesh's texture (renderer_py's texture2D, here the nearest texel of
// level 0 with clamp to edge at the interpolated UV), else its vertex colours, else grey 0.5.  Depth, coverage and
// tri_ids come straight from the key, so they equal rast_render_meshes' float-z output.
__global__ void __launch_bounds__(256)
rast_shade_kernel(const unsigned long long* __restrict__ zbuf, const MeshEntry* __restrict__ table,
                  const float* const* __restrict__ mesh_colors, const MeshTex* __restrict__ mesh_tex,
                  const int* __restrict__ mesh_ids,
                  const float* __restrict__ poses, const float* __restrict__ Ks, const float* __restrict__ colors, int n,
                  int H, int W, uint8_t* __restrict__ rgb, float* __restrict__ depth, int* __restrict__ tri_ids) {
  const long long total = (long long)n * H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long key = zbuf[i];
    if (key == 0xFFFFFFFFFFFFFFFFull) {
      depth[i] = 0.f;
      rgb[i * 3] = 0; rgb[i * 3 + 1] = 0; rgb[i * 3 + 2] = 0;
      if (tri_ids) tri_ids[i] = -1;
      continue;
    }
    depth[i] = __uint_as_float((unsigned)(key >> 32));
    const int f = (int)(unsigned)key;
    if (tri_ids) tri_ids[i] = f;
    const int px = (int)(i % W), py = (int)((i / W) % H), r = (int)(i / ((long long)H * W));
    const MeshEntry me = table[mesh_ids[r]];
    const float* P = poses + r * 12;
    const float* K = Ks + r * 9;
    float X[3], Y[3], Z[3], u[3], v[3], iz[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int vi = me.faces[f * 3 + k];
      const float x = me.verts[vi * 3], y = me.verts[vi * 3 + 1], z = me.verts[vi * 3 + 2];
      X[k] = P[0] * x + P[1] * y + P[2] * z + P[3];
      Y[k] = P[4] * x + P[5] * y + P[6] * z + P[7];
      Z[k] = P[8] * x + P[9] * y + P[10] * z + P[11];
      iz[k] = 1.0f / Z[k];
      u[k] = (K[0] * X[k] + K[1] * Y[k]) * iz[k] + K[2];
      v[k] = (K[4] * Y[k]) * iz[k] + K[5];
    }
    const float inv_area = 1.0f / ((u[1] - u[0]) * (v[2] - v[0]) - (u[2] - u[0]) * (v[1] - v[0]));
    const float sx = (float)px + 0.5f, sy = (float)py + 0.5f;
    const float w0 = ((u[1] - sx) * (v[2] - sy) - (u[2] - sx) * (v[1] - sy)) * inv_area;
    const float w1 = ((u[2] - sx) * (v[0] - sy) - (u[0] - sx) * (v[2] - sy)) * inv_area;
    const float w2 = 1.0f - w0 - w1;
    const float izp = w0 * iz[0] + w1 * iz[1] + w2 * iz[2];
    const float b[3] = {w0 * iz[0] / izp, w1 * iz[1] / izp, w2 * iz[2] / izp};
    float lx = 0.f, ly = 0.f, lz = 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {   // v_L = normalize(light - eye_pos) per vertex, light at the eye origin
      const float il = rsqrtf(X[k] * X[k] + Y[k] * Y[k] + Z[k] * Z[k]);
      lx -= b[k] * X[k] * il; ly -= b[k] * Y[k] * il; lz -= b[k] * Z[k] * il;
    }
    const float ex = X[1] - X[0], ey = Y[1] - Y[0], ez = Z[1] - Z[0];
    const float gx = X[2] - X[0], gy = Y[2] - Y[0], gz = Z[2] - Z[0];
    float nx = ey * gz - ez * gy, ny = ez * gx - ex * gz, nz = ex * gy - ey * gx;
    if (nx * X[0] + ny * Y[0] + nz * Z[0] > 0.f) { nx = -nx; ny = -ny; nz = -nz; }
    const float dot = (lx * nx + ly * ny + lz * nz) * rsqrtf(lx * lx + ly * ly + lz * lz) * rsqrtf(nx * nx + ny * ny + nz * nz);
    const float lw = fminf(0.5f + fmaxf(dot, 0.f), 1.f);
    const float* vc = mesh_colors[mesh_ids[r]];
    const MeshTex& mt = mesh_tex[mesh_ids[r]];
    float tx[3] = {0.f, 0.f, 0.f};
    const bool textured = !colors && mt.levels > 0 && mt.uvs;
    if (textured) {   // renderer_py's texture2D(u_texture, v_texcoord): nearest texel of level 0, clamp to edge
      const float* t0 = mt.uvs + me.faces[f * 3] * 2;
      const float* t1 = mt.uvs + me.faces[f * 3 + 1] * 2;
      const float* t2 = mt.uvs + me.faces[f * 3 + 2] * 2;
      const float s = b[0] * t0[0] + b[1] * t1[0] + b[2] * t2[0];
      const float t = b[0] * t0[1] + b[1] * t1[1] + b[2] * t2[1];
      const int w = mt.w[0], h = mt.h[0];
      const float xs = isfinite(s) ? fminf(fmaxf(floorf(s * (float)w), 0.f), (float)(w - 1)) : 0.f;
      const float ys = isfinite(t) ? fminf(fmaxf(floorf(t * (float)h), 0.f), (float)(h - 1)) : 0.f;
      const uint8_t* T = mt.tex + ((long long)ys * w + (long long)xs) * 3;
      tx[0] = T[0] * (1.f / 255.f); tx[1] = T[1] * (1.f / 255.f); tx[2] = T[2] * (1.f / 255.f);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float col = 0.5f;
      if (colors) col = colors[r * 3 + c];
      else if (textured) col = tx[c];
      else if (vc) col = b[0] * vc[me.faces[f * 3] * 3 + c] + b[1] * vc[me.faces[f * 3 + 1] * 3 + c] +
                         b[2] * vc[me.faces[f * 3 + 2] * 3 + c];
      rgb[i * 3 + c] = (uint8_t)fminf(fmaxf(rintf(lw * col * 255.f), 0.f), 255.f);
    }
  }
}

// ---- scene render: the n instances of one call in one image, one z-buffer (EGLRenderer.render) ---------------------
// The key's low word is the triangle's index in the concatenation of the instances' triangles in call order, so a depth
// tie between instances goes to the earlier one.  tri_off [n+1] holds each instance's first index (an unknown mesh id
// contributes no triangles); block 0 of the clear kernel fills it, before the rasteriser reads it in stream order.
__global__ void rast_scene_clear_kernel(unsigned long long* zbuf, long long npx, const MeshEntry* __restrict__ table,
                                        int n_meshes, const int* __restrict__ mesh_ids, int n, unsigned* __restrict__ tri_off) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    unsigned acc = 0;
    for (int r = 0; r < n; ++r) {
      tri_off[r] = acc;
      const int mid = mesh_ids[r];
      if (mid >= 0 && mid < n_meshes) acc += (unsigned)table[mid].F;
    }
    tri_off[n] = acc;
  }
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npx; i += (long long)gridDim.x * blockDim.x)
    zbuf[i] = 0xFFFFFFFFFFFFFFFFull;
}

__global__ void __launch_bounds__(256)
rast_scene_tri_kernel(const MeshEntry* __restrict__ table, const int* __restrict__ mesh_ids, int n_meshes, int n,
                      const float* __restrict__ poses, const float* __restrict__ K, int H, int W, float znear, float zfar,
                      const unsigned* __restrict__ tri_off, unsigned long long* __restrict__ zbuf) {
  for (int r = blockIdx.y; r < n; r += gridDim.y)
    rast_tri_one(table, mesh_ids[r], n_meshes, poses + r * 12, K, H, W, znear, zfar, zbuf, tri_off[r]);
}

// Bilinear sample of one mip level with clamp-to-edge (GL_LINEAR): texel centres at (i + 0.5) / w, row 0 at t = 0.
__device__ __forceinline__ void tex_bilinear(const MeshTex& mt, int l, float s, float t, float out[3]) {
  const int w = mt.w[l], h = mt.h[l];
  const uint8_t* T = mt.tex + mt.off[l];
  const float x = s * (float)w - 0.5f, y = t * (float)h - 0.5f;
  const float fx = floorf(x), fy = floorf(y);
  const float a = x - fx, b = y - fy;
  const int i0 = min(max((int)fx, 0), w - 1), i1 = min(max((int)fx + 1, 0), w - 1);
  const int j0 = min(max((int)fy, 0), h - 1), j1 = min(max((int)fy + 1, 0), h - 1);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float t00 = T[((long long)j0 * w + i0) * 3 + c], t10 = T[((long long)j0 * w + i1) * 3 + c];
    const float t01 = T[((long long)j1 * w + i0) * 3 + c], t11 = T[((long long)j1 * w + i1) * 3 + c];
    out[c] = ((1.f - a) * (1.f - b) * t00 + a * (1.f - b) * t10 + (1.f - a) * b * t01 + a * b * t11) * (1.f / 255.f);
  }
}

// GL_LINEAR_MIPMAP_LINEAR with GL_LINEAR magnification: lambda = log2(rho), rho the larger screen-space derivative
// length of (s w0, t h0) in level-0 texels.  lambda <= 0: level 0; lambda >= q (the last level): level q; otherwise the
// levels floor(lambda) and floor(lambda) + 1 blended by frac(lambda).
__device__ __forceinline__ void tex_sample(const MeshTex& mt, float s, float t, float dsdx, float dtdx, float dsdy,
                                           float dtdy, float out[3]) {
  if (!isfinite(s) || !isfinite(t)) { s = 0.f; t = 0.f; }
  const float W0 = (float)mt.w[0], H0 = (float)mt.h[0];
  const float rx = sqrtf((dsdx * W0) * (dsdx * W0) + (dtdx * H0) * (dtdx * H0));
  const float ry = sqrtf((dsdy * W0) * (dsdy * W0) + (dtdy * H0) * (dtdy * H0));
  const float lambda = log2f(fmaxf(rx, ry));
  const int q = mt.levels - 1;
  if (!(lambda > 0.f)) { tex_bilinear(mt, 0, s, t, out); return; }
  if (lambda >= (float)q) { tex_bilinear(mt, q, s, t, out); return; }
  const float d1 = floorf(lambda), fr = lambda - d1;
  float a[3], b[3];
  tex_bilinear(mt, (int)d1, s, t, a);
  tex_bilinear(mt, (int)d1 + 1, s, t, b);
#pragma unroll
  for (int c = 0; c < 3; ++c) out[c] = (1.f - fr) * a[c] + fr * b[c];
}

struct SceneLight {
  float pos[3], col[3];       // light position (camera frame) and colour
  float mat_diffuse[3], mat_ambient[3];
};

// Resolve: depth and pc_cam from the key with rast_resolve_kernel's arithmetic; the other outputs from the winner's
// perspective-correct barycentrics (rast_shade_kernel's arithmetic), shaded as shader_textureless_texture.{vs,frag}
// with the view matrix at identity (camera frame = world frame):
//   pc_obj = interp(x), normal = 0.5 interp(normalize(R n)) + 0.5, diff = max(dot(interp(normalize(R n)),
//   normalize(light - interp(P))), 0);  textureless: colour (diff + 0.2) light;  textured: texture (diff light
//   mat_diffuse + mat_ambient light) (the specular term is 0: with the identity view its view direction is
//   normalize(0)); every channel clamped at 1.  seg = instance index + 1.  Background: every output 0, except image
//   when a background [H,W,3] u8 is given: there image = v / 255 in f32, channels in the given order (the full-viewport
//   quad egl_renderer_v3's im2Texture draws before the models).
__global__ void __launch_bounds__(256)
rast_scene_resolve_kernel(const unsigned long long* __restrict__ zbuf, const MeshEntry* __restrict__ table,
                          const float* const* __restrict__ mesh_colors, const MeshTex* __restrict__ mesh_tex,
                          const int* __restrict__ mesh_ids, const unsigned* __restrict__ tri_off, int n,
                          const float* __restrict__ poses, const float* __restrict__ K, int H, int W, SceneLight lt,
                          const uint8_t* __restrict__ background,
                          float* __restrict__ depth, float* __restrict__ pc_cam, float* __restrict__ pc_obj,
                          float* __restrict__ normal, float* __restrict__ image, float* __restrict__ seg) {
  const long long total = (long long)H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long key = zbuf[i];
    const int px = (int)(i % W), py = (int)(i / W);
    if (key == 0xFFFFFFFFFFFFFFFFull) {
      depth[i] = 0.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        if (pc_cam) pc_cam[i * 3 + c] = 0.f;
        if (pc_obj) pc_obj[i * 3 + c] = 0.f;
        if (normal) normal[i * 3 + c] = 0.f;
        if (image) image[i * 3 + c] = background ? __fdiv_rn((float)background[i * 3 + c], 255.f) : 0.f;
      }
      if (seg) seg[i] = 0.f;
      continue;
    }
    const float z = __uint_as_float((unsigned)(key >> 32));
    depth[i] = z;
    if (pc_cam) {
      float X = 0.f, Y = 0.f;
      if (z > 0.f) {
        Y = ((float)py + 0.5f - K[5]) / K[4] * z;
        X = ((float)px + 0.5f - K[2] - K[1] * Y / z) / K[0] * z;
      }
      pc_cam[i * 3] = X; pc_cam[i * 3 + 1] = Y; pc_cam[i * 3 + 2] = z;
    }
    const unsigned g = (unsigned)key;
    int lo = 0, hi = n - 1;              // the last instance whose first triangle index is <= g
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (tri_off[mid] <= g) lo = mid; else hi = mid - 1;
    }
    const int r = lo;
    if (seg) seg[i] = (float)(r + 1);
    if (!pc_obj && !normal && !image) continue;
    const int f = (int)(g - tri_off[r]);
    const int mid = mesh_ids[r];
    const MeshEntry me = table[mid];
    const float* P = poses + r * 12;
    int vi[3];
    float X[3], Y[3], Z[3], u[3], v[3], iz[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      vi[k] = me.faces[f * 3 + k];
      const float x = me.verts[vi[k] * 3], y = me.verts[vi[k] * 3 + 1], zz = me.verts[vi[k] * 3 + 2];
      X[k] = P[0] * x + P[1] * y + P[2] * zz + P[3];
      Y[k] = P[4] * x + P[5] * y + P[6] * zz + P[7];
      Z[k] = P[8] * x + P[9] * y + P[10] * zz + P[11];
      iz[k] = 1.0f / Z[k];
      u[k] = (K[0] * X[k] + K[1] * Y[k]) * iz[k] + K[2];
      v[k] = (K[4] * Y[k]) * iz[k] + K[5];
    }
    const float inv_area = 1.0f / ((u[1] - u[0]) * (v[2] - v[0]) - (u[2] - u[0]) * (v[1] - v[0]));
    const float sx = (float)px + 0.5f, sy = (float)py + 0.5f;
    const float w0 = ((u[1] - sx) * (v[2] - sy) - (u[2] - sx) * (v[1] - sy)) * inv_area;
    const float w1 = ((u[2] - sx) * (v[0] - sy) - (u[0] - sx) * (v[2] - sy)) * inv_area;
    const float w2 = 1.0f - w0 - w1;
    const float izp = w0 * iz[0] + w1 * iz[1] + w2 * iz[2];
    const float b[3] = {w0 * iz[0] / izp, w1 * iz[1] / izp, w2 * iz[2] / izp};
    if (pc_obj) {
#pragma unroll
      for (int c = 0; c < 3; ++c)
        pc_obj[i * 3 + c] = b[0] * me.verts[vi[0] * 3 + c] + b[1] * me.verts[vi[1] * 3 + c] + b[2] * me.verts[vi[2] * 3 + c];
    }
    if (!normal && !image) continue;
    const MeshTex& mt = mesh_tex[mid];
    float N[3] = {0.f, 0.f, 0.f};
    if (mt.normals) {
#pragma unroll
      for (int k = 0; k < 3; ++k) {   // vNormalCam = normalize(R n) per vertex, interpolated, not renormalised
        const float* nk = mt.normals + vi[k] * 3;
        const float a = P[0] * nk[0] + P[1] * nk[1] + P[2] * nk[2];
        const float bb = P[4] * nk[0] + P[5] * nk[1] + P[6] * nk[2];
        const float c = P[8] * nk[0] + P[9] * nk[1] + P[10] * nk[2];
        const float d2 = a * a + bb * bb + c * c;
        const float s = d2 > 0.f ? rsqrtf(d2) : 0.f;
        N[0] += b[k] * (a * s); N[1] += b[k] * (bb * s); N[2] += b[k] * (c * s);
      }
    }
    if (normal) {
#pragma unroll
      for (int c = 0; c < 3; ++c) normal[i * 3 + c] = 0.5f * N[c] + 0.5f;
    }
    if (!image) continue;
    const float Fx = b[0] * X[0] + b[1] * X[1] + b[2] * X[2];
    const float Fy = b[0] * Y[0] + b[1] * Y[1] + b[2] * Y[2];
    const float Fz = b[0] * Z[0] + b[1] * Z[1] + b[2] * Z[2];
    float lx = lt.pos[0] - Fx, ly = lt.pos[1] - Fy, lz = lt.pos[2] - Fz;
    const float l2 = lx * lx + ly * ly + lz * lz;
    const float ls = l2 > 0.f ? rsqrtf(l2) : 0.f;
    const float diff = fmaxf(N[0] * (lx * ls) + N[1] * (ly * ls) + N[2] * (lz * ls), 0.f);
    float rgb[3];
    if (mt.levels > 0 && mt.uvs) {
      const float* t0 = mt.uvs + vi[0] * 2;
      const float* t1 = mt.uvs + vi[1] * 2;
      const float* t2 = mt.uvs + vi[2] * 2;
      const float s = b[0] * t0[0] + b[1] * t1[0] + b[2] * t2[0];
      const float t = b[0] * t0[1] + b[1] * t1[1] + b[2] * t2[1];
      // screen derivatives of the perspective-correct attribute a = sum(w_k iz_k a_k) / sum(w_k iz_k):
      // da/dx = sum(dw_k/dx iz_k (a_k - a)) / izp, with the edge-function gradients of the screen barycentrics
      const float gx[3] = {(v[1] - v[2]) * inv_area, (v[2] - v[0]) * inv_area, 0.f};
      const float gy[3] = {(u[2] - u[1]) * inv_area, (u[0] - u[2]) * inv_area, 0.f};
      const float gx2 = -(gx[0] + gx[1]), gy2 = -(gy[0] + gy[1]);
      const float dsdx = (gx[0] * iz[0] * (t0[0] - s) + gx[1] * iz[1] * (t1[0] - s) + gx2 * iz[2] * (t2[0] - s)) / izp;
      const float dtdx = (gx[0] * iz[0] * (t0[1] - t) + gx[1] * iz[1] * (t1[1] - t) + gx2 * iz[2] * (t2[1] - t)) / izp;
      const float dsdy = (gy[0] * iz[0] * (t0[0] - s) + gy[1] * iz[1] * (t1[0] - s) + gy2 * iz[2] * (t2[0] - s)) / izp;
      const float dtdy = (gy[0] * iz[0] * (t0[1] - t) + gy[1] * iz[1] * (t1[1] - t) + gy2 * iz[2] * (t2[1] - t)) / izp;
      float tx[3];
      tex_sample(mt, s, t, dsdx, dtdx, dsdy, dtdy, tx);
#pragma unroll
      for (int c = 0; c < 3; ++c) rgb[c] = tx[c] * (diff * lt.col[c] * lt.mat_diffuse[c] + lt.mat_ambient[c] * lt.col[c]);
    } else {
      const float* vc = mesh_colors[mid];
      const float cad[3] = {223.f / 255.f, 214.f / 255.f, 205.f / 255.f};   // meshutil.py:484-486, a mesh without colours
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float col = vc ? b[0] * vc[vi[0] * 3 + c] + b[1] * vc[vi[1] * 3 + c] + b[2] * vc[vi[2] * 3 + c] : cad[c];
        rgb[c] = col * (diff * lt.col[c] + 0.2f * lt.col[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) image[i * 3 + c] = fminf(rgb[c], 1.f);
  }
}

// One level of the mip chain: 2x2 box filter of the level above, rounded to nearest, (a + b + c + d + 2) >> 2 per
// channel; a source index past the last row / column is clamped to it (a dimension of 1 halves to 1).
__global__ void rast_mip_kernel(const uint8_t* __restrict__ src, int sw, int sh, uint8_t* __restrict__ dst, int dw, int dh) {
  const long long total = (long long)dw * dh;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(k % dw), j = (int)(k / dw);
    const int x0 = min(2 * i, sw - 1), x1 = min(2 * i + 1, sw - 1), y0 = min(2 * j, sh - 1), y1 = min(2 * j + 1, sh - 1);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const unsigned s = src[((long long)y0 * sw + x0) * 3 + c] + src[((long long)y0 * sw + x1) * 3 + c] +
                         src[((long long)y1 * sw + x0) * 3 + c] + src[((long long)y1 * sw + x1) * 3 + c];
      dst[k * 3 + c] = (uint8_t)((s + 2u) >> 2);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Fast depth refine, one CTA per ROI (gdrn_evaluator.py:539-561):
//   w = ||xyz|| * mask * (ren>0) * (sensor>0);  w /= sum(w);  sel = w > thresh*max(w)
//   dz = median(sensor[sel] - ren[sel]);  (y,x) = sum(w * (row, col));  ray = K^-1 (x,y,1) / z;  t += ray * dz
// weight_mode 1 (TEST.USE_COOR_Z_REFINE, gdrn_evaluator.py:528-537) replaces ||xyz|| by (R xyz)_z with the ROI's
// rotation R [n,3,3].  Those weights can be negative, and so can their sum: the reference divides by the sum first and
// takes the max over ALL pixels (zeros included) afterwards, so a negative sum takes its cut from the most negative
// raw weight.
constexpr int DR_THREADS = 1024;

// Per-stage record of depth_refine_kernel (gdrn_depth_refine_trace), device pointers, used only by the TRACE = true
// instantiation.  Entries a ROI does not reach (zero sum, empty selection) keep what the caller initialised them to.
struct DrTrace {
  float* m_lo; float* m_scale;      // [n] mask normalisation (0 and 1 unless mask_mode 1)
  float* w;                         // [n, hw*hw] raw weights before the division by the sum
  double* sum;                      // [n]
  float* max; float* min; float* cut;   // [n] reduced max / min (zero included) and the selection cut
  unsigned char* sel;               // [n, hw*hw] selected pixels
  int* count;                       // [n]
  float* median;                    // [n]
  double* centroid;                 // [n, 2] (y, x)
  double* ray;                      // [n, 3] K^-1 (x, y, 1) / z
  float* t;                         // [n, 3] the output translation
};

template <bool TRACE>
__global__ void __launch_bounds__(DR_THREADS)
depth_refine_kernel(const float* __restrict__ xyz, const float* __restrict__ mask, const float* __restrict__ sensor,
                    const float* __restrict__ ren, const float* __restrict__ Kc, float* __restrict__ trans, int hw,
                    float thresh, int mask_mode, const float* __restrict__ rot, int weight_mode, DrTrace tr) {
  extern __shared__ float sm[];  // [npix] weights, then [npow2] diffs for the sort
  const int roi = blockIdx.x;
  const int npix = hw * hw;
  float* sw = sm;
  __shared__ double red_d[32];
  __shared__ float red_f[32], red_n[32];
  __shared__ int s_count;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* X = xyz + (long long)roi * 3 * npix;
  // get_out_mask (engine/engine_utils.py:313-333) folded in: mask_mode 0 = already normalised, 1 = raw L1 output ->
  // per-ROI min-max normalisation (m - min) / (max - min), 2 = raw logits -> sigmoid (BCE / RW_BCE / dice heads)
  float m_lo = 0.f, m_scale = 1.f;
  if (mask_mode == 1) {
    float mn = INFINITY, mx = -INFINITY;
    for (int i = tid; i < npix; i += DR_THREADS) {
      const float m = mask[(long long)roi * npix + i];
      mn = fminf(mn, m); mx = fmaxf(mx, m);
    }
    for (int o = 16; o > 0; o >>= 1) {
      mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    __shared__ float red_mm[2][32];
    if (lane == 0) { red_mm[0][warp] = mn; red_mm[1][warp] = mx; }
    __syncthreads();
    mn = INFINITY; mx = -INFINITY;
    for (int k = 0; k < DR_THREADS / 32; ++k) { mn = fminf(mn, red_mm[0][k]); mx = fmaxf(mx, red_mm[1][k]); }
    m_lo = mn; m_scale = mx - mn;    // applied as a DIVISION below, like torch's (mask - min) / (max - min)
  }
  if constexpr (TRACE) { if (tid == 0) { tr.m_lo[roi] = m_lo; tr.m_scale[roi] = m_scale; } }
  // pass 1: weights, sum (double), max (and min for the signed coor-z weights)
  const float Rz0 = weight_mode == 1 ? rot[roi * 9 + 6] : 0.f, Rz1 = weight_mode == 1 ? rot[roi * 9 + 7] : 0.f,
              Rz2 = weight_mode == 1 ? rot[roi * 9 + 8] : 0.f;
  double lsum = 0.0;
  float lmax = 0.f, lmin = 0.f;
  for (int i = tid; i < npix; i += DR_THREADS) {
    const float a = X[i], b = X[npix + i], c = X[2 * npix + i];
    float mv = mask[(long long)roi * npix + i];
    if (mask_mode == 1) mv = (mv - m_lo) / m_scale;
    else if (mask_mode == 2) mv = 1.0f / (1.0f + expf(-mv));
    float wv = weight_mode == 1 ? (Rz0 * a + Rz1 * b + Rz2 * c) * mv : sqrtf(a * a + b * b + c * c) * mv;
    const float rd = ren[(long long)roi * npix + i], sd = sensor[(long long)roi * npix + i];
    if (!(rd > 0.f) || !(sd > 0.f)) wv = 0.f;
    sw[i] = wv;
    if constexpr (TRACE) tr.w[(long long)roi * npix + i] = wv;
    lsum += (double)wv;
    lmax = fmaxf(lmax, wv);
    lmin = fminf(lmin, wv);
  }
  for (int o = 16; o > 0; o >>= 1) {
    lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
    lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
    lmin = fminf(lmin, __shfl_xor_sync(0xffffffffu, lmin, o));
  }
  if (lane == 0) { red_d[warp] = lsum; red_f[warp] = lmax; red_n[warp] = lmin; }
  if (tid == 0) s_count = 0;
  __syncthreads();
  double tsum = 0.0;
  float tmax = 0.f, tmin = 0.f;
  for (int k = 0; k < DR_THREADS / 32; ++k) { tsum += red_d[k]; tmax = fmaxf(tmax, red_f[k]); tmin = fminf(tmin, red_n[k]); }
  if constexpr (TRACE) { if (tid == 0) { tr.sum[roi] = tsum; tr.max[roi] = tmax; tr.min[roi] = tmin; } }
  if (tsum == 0.0) return;  // reference: `continue` (pose unchanged)
  // w / sum is formed as (w * pre) * inv.  Below |sum| = 2^-128 the float reciprocal would overflow to inf and select
  // nothing; there the weights are scaled by pre = 2^64 and the reciprocal by 2^-64, which rounds every w / sum as the
  // unscaled product would round it if float had the exponent range.  Elsewhere pre = 1 and nothing changes.
  float inv = (float)(1.0 / tsum), pre = 1.f;
  if (isinf(inv)) { pre = 0x1p64f; inv = (float)(1.0 / (tsum * 0x1p64)); }
  // max over all pixels of w / sum: from the largest raw weight when the sum is positive, from the most negative one
  // (zeros included in both) when it is negative
  const float cut = (((weight_mode == 1 && inv < 0.f ? tmin : tmax) * pre) * inv) * thresh;
  if constexpr (TRACE) { if (tid == 0) tr.cut[roi] = cut; }
  // pass 2: weighted centroid (double) and selection of depth differences
  int npow2 = 1;
  while (npow2 < npix) npow2 <<= 1;
  float* sdiff = sm + npix;
  for (int i = tid; i < npow2; i += DR_THREADS) sdiff[i] = INFINITY;
  __syncthreads();
  double ly = 0.0, lx = 0.0;
  for (int i = tid; i < npix; i += DR_THREADS) {
    const float wn = (sw[i] * pre) * inv;
    ly += (double)wn * (double)(i / hw);
    lx += (double)wn * (double)(i % hw);
    if constexpr (TRACE) tr.sel[(long long)roi * npix + i] = wn > cut;
    if (wn > cut) {
      const int slot = atomicAdd(&s_count, 1);
      sdiff[slot] = sensor[(long long)roi * npix + i] - ren[(long long)roi * npix + i];
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    ly += __shfl_xor_sync(0xffffffffu, ly, o);
    lx += __shfl_xor_sync(0xffffffffu, lx, o);
  }
  __syncthreads();  // red_d reads above are complete
  __shared__ double red_y[32], red_x[32];
  if (lane == 0) { red_y[warp] = ly; red_x[warp] = lx; }
  __syncthreads();
  // bitonic sort of sdiff[0..npow2) ascending (INF padding sorts last)
  for (int k = 2; k <= npow2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < npow2; i += DR_THREADS) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const float a = sdiff[i], b = sdiff[ixj];
          const bool up = (i & k) == 0;
          if ((a > b) == up) { sdiff[i] = b; sdiff[ixj] = a; }
        }
      }
      __syncthreads();
    }
  }
  if (tid == 0) {
    const int cnt = s_count;
    if constexpr (TRACE) tr.count[roi] = cnt;
    if (cnt > 0) {
      // np.median: mean of the two middle elements for an even count
      const float med = (cnt & 1) ? sdiff[cnt >> 1] : 0.5f * (sdiff[(cnt >> 1) - 1] + sdiff[cnt >> 1]);
      double cy = 0.0, cx = 0.0;
      for (int k = 0; k < DR_THREADS / 32; ++k) { cy += red_y[k]; cx += red_x[k]; }
      // ray = inv(K) @ (x, y, 1), normalised by z (general 3x3 inverse in double)
      const float* K = Kc + roi * 9;
      const double a = K[0], b = K[1], c = K[2], d = K[3], e = K[4], f = K[5], g = K[6], h = K[7], i9 = K[8];
      const double det = a * (e * i9 - f * h) - b * (d * i9 - f * g) + c * (d * h - e * g);
      const double i00 = (e * i9 - f * h) / det, i01 = (c * h - b * i9) / det, i02 = (b * f - c * e) / det;
      const double i10 = (f * g - d * i9) / det, i11 = (a * i9 - c * g) / det, i12 = (c * d - a * f) / det;
      const double i20 = (d * h - e * g) / det, i21 = (b * g - a * h) / det, i22 = (a * e - b * d) / det;
      const double rx = i00 * cx + i01 * cy + i02, ry = i10 * cx + i11 * cy + i12, rz = i20 * cx + i21 * cy + i22;
      float* t = trans + roi * 3;
      t[0] = (float)((double)t[0] + rx / rz * (double)med);
      t[1] = (float)((double)t[1] + ry / rz * (double)med);
      t[2] = (float)((double)t[2] + 1.0 * (double)med);
      if constexpr (TRACE) {
        tr.median[roi] = med;
        tr.centroid[roi * 2] = cy; tr.centroid[roi * 2 + 1] = cx;
        tr.ray[roi * 3] = rx / rz; tr.ray[roi * 3 + 1] = ry / rz; tr.ray[roi * 3 + 2] = 1.0;
      }
    }
    if constexpr (TRACE) { for (int k = 0; k < 3; ++k) tr.t[roi * 3 + k] = trans[roi * 3 + k]; }
  }
}

template <bool TRACE>
int launch_depth_refine(const float* xyz, const float* mask, int mask_mode, const float* depth_sensor,
                        const float* ren_depth, const float* K_crop, const float* rot, int weight_mode, float* trans,
                        int n, int hw, float thresh, const DrTrace& tr, cudaStream_t stream) {
  int npix = hw * hw, npow2 = 1;
  while (npow2 < npix) npow2 <<= 1;
  size_t smem = (size_t)(npix + npow2) * 4;
  GDRN_OPT_IN_SMEM(depth_refine_kernel<TRACE>, 160 * 1024);
  depth_refine_kernel<TRACE><<<n, DR_THREADS, smem, stream>>>(xyz, mask, depth_sensor, ren_depth, K_crop, trans, hw,
                                                               thresh, mask_mode, rot, weight_mode, tr);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

}  // namespace

extern "C" size_t rast_scratch_bytes(int n, int H, int W) { return (size_t)n * H * W * 8; }

// ---- mesh registry: process-wide and append-only, on the device that is current at the first upload.  An id stays
// valid for the life of the process; the object that uploaded the mesh holds it (renderer.Model3D.mesh_id). -------
namespace {
struct MeshRegistry {
  int device = -1;
  int count = 0;
  int max_faces = 0;
  MeshEntry host[RAST_MAX_MESHES];
  MeshEntry* dev_table = nullptr;
  const float** dev_colors = nullptr;   // [RAST_MAX_MESHES] per-vertex RGB [V,3] f32, or null for a mesh without colours
  MeshTex* dev_tex = nullptr;           // [RAST_MAX_MESHES] normals, UVs and texture mip chain (rast_upload_mesh_tex)
};
MeshRegistry g_meshes;
}  // namespace

extern "C" int rast_upload_mesh_tex(const float* verts, int V, const int* faces, int F, const float* colors,
                                    const float* normals, const float* uvs, const uint8_t* texture, int tex_h, int tex_w) {
  // verts / faces / colors / normals / uvs / texture: host OR device pointers (cudaMemcpyDefault); the library keeps
  // its own device copy.  Returns the mesh id (>= 0) or a negative GDRN_ERR_* code.
  if (!(verts && faces && V > 0 && F > 0)) { gdrn_set_last_error(__FILE__, __LINE__, "rast_upload_mesh: empty mesh"); return GDRN_ERR_INVALID; }
  if (texture && !(uvs && tex_h > 0 && tex_w > 0)) { gdrn_set_last_error(__FILE__, __LINE__, "rast_upload_mesh_tex: a texture needs uvs and tex_h, tex_w > 0"); return GDRN_ERR_INVALID; }
  int dev = 0;
  cudaGetDevice(&dev);
  if (g_meshes.device < 0) g_meshes.device = dev;
  if (g_meshes.device != dev) { gdrn_set_last_error(__FILE__, __LINE__, "rast_upload_mesh: the mesh registry lives on another device"); return GDRN_ERR_STATE; }
  if (g_meshes.count >= RAST_MAX_MESHES) { gdrn_set_last_error(__FILE__, __LINE__, "rast_upload_mesh: registry full (1024 meshes)"); return GDRN_ERR_STATE; }
  MeshTex mt = {};
  long long tex_bytes = 0;
  if (texture) {    // level sizes: halve each dimension (floor, at least 1) until both are 1
    int w = tex_w, h = tex_h;
    for (;;) {
      mt.w[mt.levels] = w; mt.h[mt.levels] = h; mt.off[mt.levels] = tex_bytes;
      tex_bytes += (long long)w * h * 3;
      ++mt.levels;
      if (w == 1 && h == 1) break;
      if (mt.levels == RAST_MAX_MIPS) { gdrn_set_last_error(__FILE__, __LINE__, "rast_upload_mesh_tex: texture larger than 32768 texels"); return GDRN_ERR_INVALID; }
      w = w > 1 ? w / 2 : 1; h = h > 1 ? h / 2 : 1;
    }
  }
  float* dv = nullptr;
  int* df = nullptr;
  float* dc = nullptr;
  float* dn = nullptr;
  float* du = nullptr;
  uint8_t* dt = nullptr;
  cudaError_t e = cudaMalloc(&dv, (size_t)V * 12);
  if (e == cudaSuccess) e = cudaMalloc(&df, (size_t)F * 12);
  if (e == cudaSuccess) e = cudaMemcpy(dv, verts, (size_t)V * 12, cudaMemcpyDefault);
  if (e == cudaSuccess) e = cudaMemcpy(df, faces, (size_t)F * 12, cudaMemcpyDefault);
  if (e == cudaSuccess && colors) e = cudaMalloc(&dc, (size_t)V * 12);
  if (e == cudaSuccess && colors) e = cudaMemcpy(dc, colors, (size_t)V * 12, cudaMemcpyDefault);
  if (e == cudaSuccess && normals) e = cudaMalloc(&dn, (size_t)V * 12);
  if (e == cudaSuccess && normals) e = cudaMemcpy(dn, normals, (size_t)V * 12, cudaMemcpyDefault);
  if (e == cudaSuccess && uvs) e = cudaMalloc(&du, (size_t)V * 8);
  if (e == cudaSuccess && uvs) e = cudaMemcpy(du, uvs, (size_t)V * 8, cudaMemcpyDefault);
  if (e == cudaSuccess && texture) e = cudaMalloc(&dt, (size_t)tex_bytes);
  if (e == cudaSuccess && texture) e = cudaMemcpy(dt, texture, (size_t)tex_w * tex_h * 3, cudaMemcpyDefault);
  for (int l = 1; e == cudaSuccess && l < mt.levels; ++l) {
    const long long npx = (long long)mt.w[l] * mt.h[l];
    rast_mip_kernel<<<(int)((npx + 255) / 256 > 4096 ? 4096 : (npx + 255) / 256), 256>>>(
        dt + mt.off[l - 1], mt.w[l - 1], mt.h[l - 1], dt + mt.off[l], mt.w[l], mt.h[l]);
    e = cudaGetLastError();
    gdrn_count_launch(1);
  }
  if (e == cudaSuccess && mt.levels > 1) e = cudaStreamSynchronize(0);
  if (e == cudaSuccess && !g_meshes.dev_table) e = cudaMalloc(&g_meshes.dev_table, sizeof(MeshEntry) * RAST_MAX_MESHES);
  if (e == cudaSuccess && !g_meshes.dev_colors) e = cudaMalloc(&g_meshes.dev_colors, sizeof(float*) * RAST_MAX_MESHES);
  if (e == cudaSuccess && !g_meshes.dev_tex) e = cudaMalloc(&g_meshes.dev_tex, sizeof(MeshTex) * RAST_MAX_MESHES);
  if (e == cudaSuccess) {
    const int id = g_meshes.count;
    g_meshes.host[id] = MeshEntry{dv, df, V, F};
    const float* dcc = dc;
    mt.normals = dn; mt.uvs = du; mt.tex = dt;
    e = cudaMemcpy(g_meshes.dev_table + id, &g_meshes.host[id], sizeof(MeshEntry), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(g_meshes.dev_colors + id, &dcc, sizeof(float*), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(g_meshes.dev_tex + id, &mt, sizeof(MeshTex), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
      g_meshes.count = id + 1;
      if (F > g_meshes.max_faces) g_meshes.max_faces = F;
      return id;
    }
  }
  (void)cudaGetLastError();
  cudaFree(dv); cudaFree(df); cudaFree(dc); cudaFree(dn); cudaFree(du); cudaFree(dt);
  gdrn_set_last_error(__FILE__, __LINE__, cudaGetErrorString(e));
  return GDRN_ERR_CUDA;
}

extern "C" int rast_upload_mesh_ex(const float* verts, int V, const int* faces, int F, const float* colors) {
  return rast_upload_mesh_tex(verts, V, faces, F, colors, nullptr, nullptr, nullptr, 0, 0);
}

extern "C" int rast_upload_mesh(const float* verts, int V, const int* faces, int F) {
  return rast_upload_mesh_ex(verts, V, faces, F, nullptr);
}

extern "C" int rast_mesh_count(void) { return g_meshes.count; }

extern "C" int rast_render_meshes(const int* mesh_ids, const float* poses, const float* Ks, int n, int H, int W,
                                  float znear, float zfar, int quantize_bits, float* depth, float* xyz_cam,
                                  unsigned long long* zbuf_scratch, void* stream) {
  GDRN_REQUIRE(mesh_ids && poses && Ks && depth && zbuf_scratch, "rast_render_meshes: null argument");
  GDRN_REQUIRE(n > 0 && H > 0 && W > 0, "rast_render_meshes: empty input");
  GDRN_REQUIRE(g_meshes.count > 0, "rast_render_meshes: no mesh uploaded (rast_upload_mesh)");
  GDRN_REQUIRE(quantize_bits == 0 || quantize_bits == 16 || quantize_bits == 24 || quantize_bits == 32,
               "rast: quantize_bits must be 0, 16, 24 or 32");
  GDRN_REQUIRE(znear > 0.f && zfar > znear, "rast: need 0 < znear < zfar");
  cudaStream_t st = (cudaStream_t)stream;
  const long long npx = (long long)n * H * W;
  int blocks = (int)((npx + 255) / 256 > 4096 ? 4096 : (npx + 255) / 256);
  rast_clear_kernel<<<blocks, 256, 0, st>>>(zbuf_scratch, npx);
  rast_tri_multi_kernel<<<dim3((g_meshes.max_faces + 255) / 256, n < 65535 ? n : 65535), 256, 0, st>>>(
      g_meshes.dev_table, mesh_ids, g_meshes.count, n, poses, Ks, H, W, znear, zfar, zbuf_scratch);
  rast_resolve_kernel<<<blocks, 256, 0, st>>>(zbuf_scratch, Ks, n, H, W, znear, zfar, quantize_bits, depth, xyz_cam);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(3);
  return GDRN_OK;
}

extern "C" int rast_render_meshes_rgb(const int* mesh_ids, const float* poses, const float* Ks, const float* colors, int n,
                                      int H, int W, float znear, float zfar, uint8_t* rgb, float* depth, int* tri_ids,
                                      unsigned long long* zbuf_scratch, void* stream) {
  GDRN_REQUIRE(mesh_ids && poses && Ks && rgb && depth && zbuf_scratch, "rast_render_meshes_rgb: null argument");
  GDRN_REQUIRE(n > 0 && H > 0 && W > 0, "rast_render_meshes_rgb: empty input");
  GDRN_REQUIRE(g_meshes.count > 0, "rast_render_meshes_rgb: no mesh uploaded (rast_upload_mesh)");
  GDRN_REQUIRE(znear > 0.f && zfar > znear, "rast: need 0 < znear < zfar");
  cudaStream_t st = (cudaStream_t)stream;
  const long long npx = (long long)n * H * W;
  int blocks = (int)((npx + 255) / 256 > 4096 ? 4096 : (npx + 255) / 256);
  rast_clear_kernel<<<blocks, 256, 0, st>>>(zbuf_scratch, npx);
  rast_tri_multi_kernel<<<dim3((g_meshes.max_faces + 255) / 256, n < 65535 ? n : 65535), 256, 0, st>>>(
      g_meshes.dev_table, mesh_ids, g_meshes.count, n, poses, Ks, H, W, znear, zfar, zbuf_scratch);
  rast_shade_kernel<<<blocks, 256, 0, st>>>(zbuf_scratch, g_meshes.dev_table, g_meshes.dev_colors, g_meshes.dev_tex, mesh_ids, poses, Ks, colors,
                                            n, H, W, rgb, depth, tri_ids);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(3);
  return GDRN_OK;
}

// zbuf [H*W] u64, then the per-instance first-triangle table [n_inst + 1] u32
extern "C" size_t rast_scene_scratch_bytes(int n_inst, int H, int W) {
  return (size_t)H * W * 8 + (((size_t)n_inst + 1) * 4 + 7) / 8 * 8;
}

extern "C" int rast_render_scene_bg(const int* mesh_ids, const float* poses, int n_inst, const float* K, int H, int W,
                                    float znear, float zfar, const float* light, const uint8_t* background, float* depth,
                                    float* pc_cam, float* pc_obj, float* normal, float* image, float* seg, void* scratch,
                                    void* stream) {
  GDRN_REQUIRE(K && light && depth && scratch && (n_inst == 0 || (mesh_ids && poses)), "rast_render_scene: null argument");
  GDRN_REQUIRE(n_inst >= 0 && H > 0 && W > 0, "rast_render_scene: empty input");
  GDRN_REQUIRE(n_inst > 0 || background, "rast_render_scene: no instance and no background");
  GDRN_REQUIRE(n_inst == 0 || g_meshes.count > 0, "rast_render_scene: no mesh uploaded (rast_upload_mesh)");
  GDRN_REQUIRE(znear > 0.f && zfar > znear, "rast: need 0 < znear < zfar");
  SceneLight lt;
  for (int c = 0; c < 3; ++c) {
    lt.pos[c] = light[c]; lt.col[c] = light[3 + c]; lt.mat_diffuse[c] = light[6 + c]; lt.mat_ambient[c] = light[9 + c];
  }
  cudaStream_t st = (cudaStream_t)stream;
  const long long npx = (long long)H * W;
  unsigned long long* zbuf = (unsigned long long*)scratch;
  unsigned* tri_off = (unsigned*)(zbuf + npx);
  int blocks = (int)((npx + 255) / 256 > 4096 ? 4096 : (npx + 255) / 256);
  rast_scene_clear_kernel<<<blocks, 256, 0, st>>>(zbuf, npx, g_meshes.dev_table, g_meshes.count, mesh_ids, n_inst, tri_off);
  if (n_inst > 0)
    rast_scene_tri_kernel<<<dim3((g_meshes.max_faces + 255) / 256, n_inst < 65535 ? n_inst : 65535), 256, 0, st>>>(
        g_meshes.dev_table, mesh_ids, g_meshes.count, n_inst, poses, K, H, W, znear, zfar, tri_off, zbuf);
  rast_scene_resolve_kernel<<<blocks, 256, 0, st>>>(zbuf, g_meshes.dev_table, g_meshes.dev_colors, g_meshes.dev_tex,
                                                    mesh_ids, tri_off, n_inst, poses, K, H, W, lt, background, depth,
                                                    pc_cam, pc_obj, normal, image, seg);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(n_inst > 0 ? 3 : 2);
  return GDRN_OK;
}

extern "C" int rast_render_scene(const int* mesh_ids, const float* poses, int n_inst, const float* K, int H, int W,
                                 float znear, float zfar, const float* light, float* depth, float* pc_cam, float* pc_obj,
                                 float* normal, float* image, float* seg, void* scratch, void* stream) {
  GDRN_REQUIRE(mesh_ids && poses && K && light && depth && scratch, "rast_render_scene: null argument");
  GDRN_REQUIRE(n_inst > 0 && H > 0 && W > 0, "rast_render_scene: empty input");
  return rast_render_scene_bg(mesh_ids, poses, n_inst, K, H, W, znear, zfar, light, nullptr, depth, pc_cam, pc_obj,
                              normal, image, seg, scratch, stream);
}

extern "C" int gdrn_depth_refine_step(const float* xyz, const float* mask, int mask_mode, const float* depth_sensor,
                                      const float* ren_depth, const float* K_crop, const float* rot, int weight_mode,
                                      float* trans, int n, int hw, float thresh, void* stream) {
  GDRN_REQUIRE(xyz && mask && depth_sensor && ren_depth && K_crop && trans, "depth_refine: null argument");
  GDRN_REQUIRE(mask_mode >= 0 && mask_mode <= 2, "depth_refine: mask_mode must be 0 (normalised), 1 (raw L1) or 2 (logits)");
  GDRN_REQUIRE(weight_mode == 0 || weight_mode == 1, "depth_refine: weight_mode must be 0 (||xyz||) or 1 (coor-z)");
  GDRN_REQUIRE(weight_mode == 0 || rot, "depth_refine: the coor-z weighting needs the rotations");
  GDRN_REQUIRE(n > 0 && hw > 0 && hw <= 128, "depth_refine: need 0 < hw <= 128");
  return launch_depth_refine<false>(xyz, mask, mask_mode, depth_sensor, ren_depth, K_crop, rot, weight_mode, trans, n,
                                    hw, thresh, DrTrace{}, (cudaStream_t)stream);
}

extern "C" int gdrn_depth_refine_trace(const float* xyz, const float* mask, int mask_mode, const float* depth_sensor,
                                       const float* ren_depth, const float* K_crop, const float* rot, int weight_mode,
                                       float* trans, int n, int hw, float thresh, float* tr_m_lo, float* tr_m_scale,
                                       float* tr_w, double* tr_sum, float* tr_max, float* tr_min, float* tr_cut,
                                       unsigned char* tr_sel, int* tr_count, float* tr_median, double* tr_centroid,
                                       double* tr_ray, float* tr_t, void* stream) {
  GDRN_REQUIRE(xyz && mask && depth_sensor && ren_depth && K_crop && trans, "depth_refine_trace: null argument");
  GDRN_REQUIRE(tr_m_lo && tr_m_scale && tr_w && tr_sum && tr_max && tr_min && tr_cut && tr_sel && tr_count && tr_median &&
               tr_centroid && tr_ray && tr_t, "depth_refine_trace: null trace buffer");
  GDRN_REQUIRE(mask_mode >= 0 && mask_mode <= 2, "depth_refine: mask_mode must be 0 (normalised), 1 (raw L1) or 2 (logits)");
  GDRN_REQUIRE(weight_mode == 0 || weight_mode == 1, "depth_refine: weight_mode must be 0 (||xyz||) or 1 (coor-z)");
  GDRN_REQUIRE(weight_mode == 0 || rot, "depth_refine: the coor-z weighting needs the rotations");
  GDRN_REQUIRE(n > 0 && hw > 0 && hw <= 128, "depth_refine: need 0 < hw <= 128");
  const DrTrace tr = {tr_m_lo, tr_m_scale, tr_w, tr_sum, tr_max, tr_min, tr_cut, tr_sel, tr_count, tr_median,
                      tr_centroid, tr_ray, tr_t};
  return launch_depth_refine<true>(xyz, mask, mask_mode, depth_sensor, ren_depth, K_crop, rot, weight_mode, trans, n,
                                   hw, thresh, tr, (cudaStream_t)stream);
}
