// mesh.cu -- mesh extraction from the rendered expected depth (ours; DESIGN.md section 1, "Mesh extraction"): TSDF fusion of
// batches of views into a dense lattice, and marching tetrahedra on the Freudenthal (Kuhn) subdivision of its cells, written in
// a canonical order so that the mesh is a plain function of the volume.
//
// The lattice has nx x ny x nz points, x fastest; point (i, j, k) sits at origin + (i h, j h, k h).  Cell a is the cube with
// lower corner a; cube corner c (bit 0 = +x, bit 1 = +y, bit 2 = +z) is a + (c & 1, c >> 1 & 1, c >> 2 & 1).
//
// Integration: one thread per lattice point walks the views in index order (no atomics: bit-reproducible, and one batch of V
// views gives the bits of V single-view launches); every step is one correctly rounded fp32 operation in the order of
// DESIGN.md, with __fmul_rn / __fadd_rn / __fdiv_rn where contraction would change bits.
//
// Extraction: lgs_mesh_count writes, per lattice point, the mask of its 7 edges a -> a + d that carry a vertex, its vertex
// count and the triangle count of the cell it is the lower corner of; the caller scans the counts into int64 offsets, and
// lgs_mesh_emit writes the vertices in (point, edge direction) order and the triangles in (cell, tetrahedron, triangle) order.
#include "common.cuh"

namespace {

constexpr int NT = 256;
constexpr int CAM_CHUNK = 64;                // views staged in shared memory at a time
constexpr int CAM_FLOATS = 32;               // view (row-vector, 16) then proj (16)

// Edge directions 0..6 as cube-corner masks: x, y, z, x+y, x+z, y+z, x+y+z.
__device__ __forceinline__ int dir_mask(int d) { return d < 3 ? 1 << d : (d == 3 ? 3 : d + 1); }
// and back: the direction of the edge from corner c to corner c | m
__device__ __forceinline__ int mask_dir(int m) { return m == 1 ? 0 : m == 2 ? 1 : m == 4 ? 2 : m == 3 ? 3 : m - 1; }

// The 6 tetrahedra 0 -> e_p1 -> e_p1 + e_p2 -> (1,1,1), one per permutation p of the axes in lexicographic order, as cube
// corners (nibble v of the word: {0,1,3,7}, {0,1,5,7}, {0,2,3,7}, {0,2,6,7}, {0,4,5,7}, {0,4,6,7}; no array, so no local
// memory), and the sign of each permutation (= the orientation of the tetrahedron).
__device__ __forceinline__ int tet_corner(int t, int v)
{
    const unsigned w = t == 0 ? 0x7310u : t == 1 ? 0x7510u : t == 2 ? 0x7320u : t == 3 ? 0x7620u : t == 4 ? 0x7540u : 0x7640u;
    return (int)((w >> (4 * v)) & 15u);
}
__device__ __forceinline__ int tet_sign(int t) { return (t == 0 || t == 3 || t == 4) ? 1 : -1; }

template <bool COLOR>
__global__ void __launch_bounds__(NT) tsdf_integrate_kernel(float* __restrict__ tsdf, float* __restrict__ weight, float* __restrict__ color,
                                                            int nx, int ny, unsigned N, float ox, float oy, float oz, float h, float trunc,
                                                            const float* __restrict__ D, const float* __restrict__ T,
                                                            const float* __restrict__ rgb, const float* __restrict__ view,
                                                            const float* __restrict__ proj, int V, int H, int W, float alpha_min,
                                                            float depth_far)
{
    __shared__ float s_cam[CAM_CHUNK][CAM_FLOATS];
    const unsigned nxy = (unsigned)nx * (unsigned)ny;
    const unsigned idx = blockIdx.x * NT + threadIdx.x;
    const bool live = idx < N;
    const unsigned k = idx / nxy, r = idx - k * nxy, j = r / (unsigned)nx, i = r - j * (unsigned)nx;
    const float p0 = __fadd_rn(ox, __fmul_rn((float)i, h)), p1 = __fadd_rn(oy, __fmul_rn((float)j, h)),
                p2 = __fadd_rn(oz, __fmul_rn((float)k, h));
    float ts = 1.0f, w = 0.0f, c[3] = {0.0f, 0.0f, 0.0f};
    if (live) {
        ts = tsdf[idx];
        w = weight[idx];
        if (COLOR)
#pragma unroll
            for (int ch = 0; ch < 3; ch++) c[ch] = color[(size_t)ch * N + idx];
    }
    const float Wf = (float)W, Hf = (float)H, cx = __fmul_rn(Wf, 0.5f), cy = __fmul_rn(Hf, 0.5f);
    const size_t HW = (size_t)H * W;
    for (int base = 0; base < V; base += CAM_CHUNK) {
        const int nb = min(CAM_CHUNK, V - base);
        __syncthreads();
        for (int e = threadIdx.x; e < nb * CAM_FLOATS; e += NT) {
            const int v = e / CAM_FLOATS, q = e % CAM_FLOATS;
            s_cam[v][q] = q < 16 ? view[(size_t)(base + v) * 16 + q] : proj[(size_t)(base + v) * 16 + (q - 16)];
        }
        __syncthreads();
        if (!live) continue;
        for (int vv = 0; vv < nb; vv++) {
            const float* m = s_cam[vv];
            // 1. view-space position p~ V, as filter_3d_kernel's z_v
            const float z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(p0, m[2]), __fmul_rn(p1, m[6])), __fmul_rn(p2, m[10])), m[14]);
            if (!(z > 0.01f)) continue;
            const float x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(p0, m[0]), __fmul_rn(p1, m[4])), __fmul_rn(p2, m[8])), m[12]);
            const float y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(p0, m[1]), __fmul_rn(p1, m[5])), __fmul_rn(p2, m[9])), m[13]);
            // 2. pixel coordinates, the inverse of lgs_depth_normal's ray ((u + 0.5 - W/2) / fx, (v + 0.5 - H/2) / fy, 1)
            const float fx = __fmul_rn(__fmul_rn(m[16], Wf), 0.5f), fy = __fmul_rn(__fmul_rn(m[21], Hf), 0.5f);
            const float u = __fadd_rn(__fmul_rn(__fdiv_rn(x, z), fx), cx);
            const float wv = __fadd_rn(__fmul_rn(__fdiv_rn(y, z), fy), cy);
            // 3. the pixel (floor(u), floor(wv)) inside the image (NaN fails every comparison)
            if (!(u >= 0.0f && u < Wf && wv >= 0.0f && wv < Hf)) continue;
            const size_t pix = (size_t)(int)wv * W + (int)u, o = (size_t)(base + vv) * HW + pix;
            // 4. alpha and the expected depth
            const float a = __fsub_rn(1.0f, T[o]);
            if (!(a > alpha_min)) continue;
            const float ed = __fdiv_rn(D[o], a);
            if (ed > depth_far) continue;
            // 5. truncated signed distance along the optical axis
            const float sdf = __fsub_rn(ed, z);
            if (sdf < -trunc) continue;
            const float t = fminf(1.0f, __fdiv_rn(sdf, trunc));
            // 6. running weighted means
            const float w1 = __fadd_rn(w, 1.0f);
            ts = __fdiv_rn(__fadd_rn(__fmul_rn(ts, w), t), w1);
            if (COLOR) {
                const size_t oc = (size_t)(base + vv) * 3 * HW + pix;
#pragma unroll
                for (int ch = 0; ch < 3; ch++) {
                    const float e = fminf(1.0f, fmaxf(0.0f, __fdiv_rn(rgb[oc + ch * HW], a)));
                    c[ch] = __fdiv_rn(__fadd_rn(__fmul_rn(c[ch], w), e), w1);
                }
            }
            w = w1;
        }
    }
    if (live) {
        tsdf[idx] = ts;
        weight[idx] = w;
        if (COLOR)
#pragma unroll
            for (int ch = 0; ch < 3; ch++) color[(size_t)ch * N + idx] = c[ch];
    }
}

struct Lattice {
    int nx, ny, nz;
    unsigned nxy, N;
    __device__ __forceinline__ void coords(unsigned idx, int& i, int& j, int& k) const
    {
        k = (int)(idx / nxy);
        const unsigned r = idx - (unsigned)k * nxy;
        j = (int)(r / (unsigned)nx);
        i = (int)(r - (unsigned)j * nx);
    }
    // linear offset of cube corner c
    __device__ __forceinline__ unsigned corner(int c) const { return (c & 1) + ((c >> 1) & 1) * (unsigned)nx + ((c >> 2) & 1) * nxy; }
};

// Per lattice point a: the weight test of its 3x3x3 neighbourhood gives the validity of the 8 cells that have a as a corner;
// edge a -> a + d belongs to the cells with lower corner a - o, o_axis = 0 on the axes of d and o_axis in {0, 1} elsewhere.
__global__ void __launch_bounds__(NT) mesh_count_kernel(const float* __restrict__ tsdf, const float* __restrict__ weight, Lattice L,
                                                        float weight_min, uint8_t* __restrict__ vmask, uint8_t* __restrict__ vcount,
                                                        uint8_t* __restrict__ fcount)
{
    const unsigned idx = blockIdx.x * NT + threadIdx.x;
    if (idx >= L.N) return;
    int i, j, k;
    L.coords(idx, i, j, k);
    unsigned ok = 0;                      // bit (dx+1) + 3 (dy+1) + 9 (dz+1): weight >= weight_min at a + (dx, dy, dz)
#pragma unroll
    for (int dz = -1; dz <= 1; dz++)
#pragma unroll
        for (int dy = -1; dy <= 1; dy++)
#pragma unroll
            for (int dx = -1; dx <= 1; dx++) {
                const int x = i + dx, y = j + dy, z = k + dz;
                if (x < 0 || x >= L.nx || y < 0 || y >= L.ny || z < 0 || z >= L.nz) continue;
                const long long q = (long long)idx + dx + (long long)dy * L.nx + (long long)dz * L.nxy;
                if (weight[q] >= weight_min) ok |= 1u << ((dx + 1) + 3 * (dy + 1) + 9 * (dz + 1));
            }
    unsigned cells = 0;                   // bit (ox+1) | (oy+1) << 1 | (oz+1) << 2: the cell with lower corner a + o is valid
#pragma unroll
    for (int c = 0; c < 8; c++) {
        const int ox = (c & 1) - 1, oy = ((c >> 1) & 1) - 1, oz = ((c >> 2) & 1) - 1;
        unsigned need = 0;
#pragma unroll
        for (int d = 0; d < 8; d++)
            need |= 1u << ((ox + (d & 1) + 1) + 3 * (oy + ((d >> 1) & 1) + 1) + 9 * (oz + ((d >> 2) & 1) + 1));
        if ((ok & need) == need) cells |= 1u << c;
    }
    const float ta = tsdf[idx];
    unsigned vm = 0;
#pragma unroll
    for (int d = 0; d < 7; d++) {
        const int m = dir_mask(d);
        unsigned owners = 0;              // the cells containing edge d: (c & m) == m
#pragma unroll
        for (int c = 0; c < 8; c++)
            if ((c & m) == m) owners |= 1u << c;
        if (!(cells & owners)) continue;
        const float tb = tsdf[idx + L.corner(m)];
        if ((ta < 0.0f) != (tb < 0.0f)) vm |= 1u << d;
    }
    unsigned fc = 0;
    if (cells & 0x80u) {                  // the cell with lower corner a
        unsigned in = 0;
#pragma unroll
        for (int c = 0; c < 8; c++)
            if (tsdf[idx + L.corner(c)] < 0.0f) in |= 1u << c;
#pragma unroll
        for (int t = 0; t < 6; t++) {
            int n = 0;
#pragma unroll
            for (int v = 0; v < 4; v++) n += (in >> tet_corner(t, v)) & 1;
            fc += n == 2 ? 2 : (n == 1 || n == 3) ? 1 : 0;
        }
    }
    vmask[idx] = (uint8_t)vm;
    vcount[idx] = (uint8_t)__popc(vm);
    fcount[idx] = (uint8_t)fc;
}

template <bool COLOR>
__global__ void __launch_bounds__(NT) mesh_vertices_kernel(const float* __restrict__ tsdf, const float* __restrict__ color, Lattice L,
                                                           float ox, float oy, float oz, float h, const uint8_t* __restrict__ vmask,
                                                           const long long* __restrict__ vert_end, float* __restrict__ vertices,
                                                           uint8_t* __restrict__ vcolors)
{
    const unsigned idx = blockIdx.x * NT + threadIdx.x;
    if (idx >= L.N) return;
    const unsigned m = vmask[idx];
    if (!m) return;
    int i, j, k;
    L.coords(idx, i, j, k);
    long long out = vert_end[idx] - __popc(m);
    const float ta = tsdf[idx];
    const float pa[3] = {__fadd_rn(ox, __fmul_rn((float)i, h)), __fadd_rn(oy, __fmul_rn((float)j, h)), __fadd_rn(oz, __fmul_rn((float)k, h))};
#pragma unroll
    for (int d = 0; d < 7; d++) {
        if (!((m >> d) & 1)) continue;
        const int dm = dir_mask(d);
        const unsigned q = idx + L.corner(dm);
        const float s = __fdiv_rn(ta, __fsub_rn(ta, tsdf[q]));
        const float pb[3] = {__fadd_rn(ox, __fmul_rn((float)(i + (dm & 1)), h)), __fadd_rn(oy, __fmul_rn((float)(j + ((dm >> 1) & 1)), h)),
                             __fadd_rn(oz, __fmul_rn((float)(k + ((dm >> 2) & 1)), h))};
#pragma unroll
        for (int ax = 0; ax < 3; ax++) vertices[out * 3 + ax] = __fadd_rn(pa[ax], __fmul_rn(s, __fsub_rn(pb[ax], pa[ax])));
        if (COLOR) {
#pragma unroll
            for (int ch = 0; ch < 3; ch++) {
                const float ca = color[(size_t)ch * L.N + idx], cb = color[(size_t)ch * L.N + q];
                const float cv = __fadd_rn(ca, __fmul_rn(s, __fsub_rn(cb, ca)));
                vcolors[out * 3 + ch] = (uint8_t)min(255, max(0, __float2int_rn(__fmul_rn(cv, 255.0f))));
            }
        }
        out++;
    }
}

// Index of the vertex on the edge from cube corner ca to cube corner cb (ca a subset of cb) of the cell with lower corner idx.
__device__ __forceinline__ int edge_vertex(const Lattice& L, unsigned idx, int ca, int cb, const uint8_t* __restrict__ vmask,
                                           const long long* __restrict__ vert_end)
{
    if ((ca & cb) != ca) { const int s = ca; ca = cb; cb = s; }
    const unsigned q = idx + L.corner(ca);
    const unsigned m = vmask[q];
    const int d = mask_dir(ca ^ cb);
    return (int)(vert_end[q] - __popc(m) + __popc(m & ((1u << d) - 1u)));
}

// One tetrahedron's triangles; a tetrahedron (P0, P1, P2, P3) of positive orientation has face (P1, P2, P3) wound with its
// right-hand normal away from P0, so each case below is wound toward the corners with tsdf >= 0.
__global__ void __launch_bounds__(NT) mesh_faces_kernel(const float* __restrict__ tsdf, Lattice L, const uint8_t* __restrict__ vmask,
                                                        const uint8_t* __restrict__ fcount, const long long* __restrict__ vert_end,
                                                        const long long* __restrict__ face_end, int* __restrict__ faces)
{
    const unsigned idx = blockIdx.x * NT + threadIdx.x;
    if (idx >= L.N) return;
    const int fc = fcount[idx];
    if (!fc) return;
    long long out = face_end[idx] - fc;
    unsigned in = 0;
#pragma unroll
    for (int c = 0; c < 8; c++)
        if (tsdf[idx + L.corner(c)] < 0.0f) in |= 1u << c;
    auto E = [&](int t, int x, int y) { return edge_vertex(L, idx, tet_corner(t, x), tet_corner(t, y), vmask, vert_end); };
    auto put = [&](int v0, int v1, int v2) {
        faces[out * 3] = v0; faces[out * 3 + 1] = v1; faces[out * 3 + 2] = v2;
        out++;
    };
#pragma unroll
    for (int t = 0; t < 6; t++) {
        int s = 0, n = 0;
#pragma unroll
        for (int v = 0; v < 4; v++) {
            const int b = (in >> tet_corner(t, v)) & 1;
            s |= b << v;
            n += b;
        }
        if (n == 0 || n == 4) continue;
        if (n == 1 || n == 3) {
            // the lone corner a (inside for n = 1, outside for n = 3) and the others b < c < d; (a, b, c, d) has parity (-1)^a
            const int a = __ffs(n == 1 ? s : (~s & 15)) - 1;
            const int b = a == 0 ? 1 : 0, c = a <= 1 ? 2 : 1, d = a <= 2 ? 3 : 2;
            // n = 1: wind away from a when (a, b, c, d) is positive; n = 3: toward a, i.e. the other way round
            const bool pos = (tet_sign(t) * ((a & 1) ? -1 : 1) > 0) == (n == 1);
            if (pos) put(E(t, a, b), E(t, a, c), E(t, a, d));
            else put(E(t, a, b), E(t, a, d), E(t, a, c));
        } else {
            // inside a < b, outside c < d; the quad (a,c) (a,d) (b,d) (b,c) is split along (a,c)-(b,d)
            const int a = __ffs(s) - 1, b = __ffs(s & (s - 1)) - 1;
            const int o = ~s & 15;
            const int c = __ffs(o) - 1, d = __ffs(o & (o - 1)) - 1;
            const bool odd = (s == 5 || s == 10);                 // inside {0,2} or {1,3}: (a, b, c, d) is an odd permutation
            const int ac = E(t, a, c), ad = E(t, a, d), bd = E(t, b, d), bc = E(t, b, c);
            if (tet_sign(t) * (odd ? -1 : 1) > 0) { put(ac, ad, bd); put(ac, bd, bc); }
            else { put(ac, bd, ad); put(ac, bc, bd); }
        }
    }
}

int lattice_of(int nx, int ny, int nz, Lattice& L, const char* who)
{
    LGS_REQUIRE(nx >= 1 && ny >= 1 && nz >= 1, "%s: bad lattice %d x %d x %d", who, nx, ny, nz);
    const long long n = (long long)nx * ny * nz;
    LGS_REQUIRE(n < (1ll << 31), "%s: %lld lattice points exceed 2^31 - 1", who, n);
    L = {nx, ny, nz, (unsigned)nx * (unsigned)ny, (unsigned)n};
    return LGS_OK;
}

}  // namespace

extern "C" int lgs_tsdf_integrate(float* tsdf, float* weight, float* color, int nx, int ny, int nz, float ox, float oy, float oz,
                                  float voxel_size, float sdf_trunc, const float* depth, const float* trans, const float* rgb,
                                  const float* view, const float* proj, int V, int H, int W, float alpha_min, float depth_far,
                                  void* stream)
{
    Lattice L;
    if (int e = lattice_of(nx, ny, nz, L, "tsdf_integrate")) return e;
    LGS_REQUIRE(tsdf != nullptr && weight != nullptr, "tsdf_integrate: null tsdf or weight");
    LGS_REQUIRE(depth != nullptr && trans != nullptr && view != nullptr && proj != nullptr,
                "tsdf_integrate: null depth, transmittance, view or projection");
    LGS_REQUIRE((color == nullptr) == (rgb == nullptr), "tsdf_integrate: the colour volume and the rgb images come together");
    LGS_REQUIRE(V >= 1 && H >= 1 && W >= 1, "tsdf_integrate: bad batch [%d, %d, %d]", V, H, W);
    LGS_REQUIRE(voxel_size > 0.0f && sdf_trunc > 0.0f, "tsdf_integrate: voxel_size = %g and sdf_trunc = %g must be positive",
                (double)voxel_size, (double)sdf_trunc);
    LGS_REQUIRE(alpha_min >= 0.0f && alpha_min < 1.0f, "tsdf_integrate: alpha_min = %g outside [0, 1)", (double)alpha_min);
    const unsigned blocks = (L.N + NT - 1) / NT;
    cudaStream_t st = (cudaStream_t)stream;
    lgs_with_flags([&](auto col) {
        tsdf_integrate_kernel<col><<<blocks, NT, 0, st>>>(tsdf, weight, color, nx, ny, L.N, ox, oy, oz, voxel_size, sdf_trunc, depth, trans,
                                                          rgb, view, proj, V, H, W, alpha_min, depth_far);
        return LGS_OK;
    }, color != nullptr);
    LGS_CHECK_LAUNCH("tsdf_integrate_kernel");
    return LGS_OK;
}

extern "C" int lgs_mesh_count(const float* tsdf, const float* weight, int nx, int ny, int nz, float weight_min, unsigned char* vmask,
                              unsigned char* vcount, unsigned char* fcount, void* stream)
{
    Lattice L;
    if (int e = lattice_of(nx, ny, nz, L, "mesh_count")) return e;
    LGS_REQUIRE(tsdf != nullptr && weight != nullptr && vmask != nullptr && vcount != nullptr && fcount != nullptr,
                "mesh_count: null argument");
    mesh_count_kernel<<<(L.N + NT - 1) / NT, NT, 0, (cudaStream_t)stream>>>(tsdf, weight, L, weight_min, vmask, vcount, fcount);
    LGS_CHECK_LAUNCH("mesh_count_kernel");
    return LGS_OK;
}

extern "C" int lgs_mesh_emit(const float* tsdf, const float* color, int nx, int ny, int nz, float ox, float oy, float oz, float voxel_size,
                             const unsigned char* vmask, const unsigned char* fcount, const long long* vert_end, const long long* face_end,
                             long long n_vertices, long long n_faces, float* vertices, int* faces, unsigned char* vcolors, void* stream)
{
    LGS_REQUIRE(n_vertices >= 0 && n_vertices < (1ll << 31) && n_faces >= 0 && n_faces < (1ll << 31),
                "mesh_emit: %lld vertices and %lld faces; int32 indices need both below 2^31", n_vertices, n_faces);
    Lattice L;
    if (int e = lattice_of(nx, ny, nz, L, "mesh_emit")) return e;
    LGS_REQUIRE(tsdf != nullptr && vmask != nullptr && fcount != nullptr && vert_end != nullptr && face_end != nullptr,
                "mesh_emit: null argument");
    if (n_vertices == 0 && n_faces == 0) return LGS_OK;       // empty outputs may have null data pointers
    LGS_REQUIRE((color == nullptr) == (vcolors == nullptr), "mesh_emit: the colour volume and the vertex colours come together");
    LGS_REQUIRE(vertices != nullptr && faces != nullptr, "mesh_emit: null output");
    const unsigned blocks = (L.N + NT - 1) / NT;
    cudaStream_t st = (cudaStream_t)stream;
    lgs_with_flags([&](auto col) {
        mesh_vertices_kernel<col><<<blocks, NT, 0, st>>>(tsdf, color, L, ox, oy, oz, voxel_size, vmask, vert_end, vertices, vcolors);
        return LGS_OK;
    }, color != nullptr);
    LGS_CHECK_LAUNCH("mesh_vertices_kernel");
    mesh_faces_kernel<<<blocks, NT, 0, st>>>(tsdf, L, vmask, fcount, vert_end, face_end, faces);
    LGS_CHECK_LAUNCH("mesh_faces_kernel");
    return LGS_OK;
}
