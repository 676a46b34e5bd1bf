// TSDF fusion of rendered depth (and colour) into a dense voxel grid, and marching-cubes extraction of a welded,
// coloured triangle mesh.  The semantics are stated in include/r3dg_b200.h (r3dg_tsdf_*) and tsdf.py.
//   integrate: ONE kernel, one thread per grid point, consecutive threads on consecutive k (the fastest axis), so the
//              tsdf / weight / color reads and writes are coalesced.  The call's V view matrices sit in shared memory
//              and the intrinsics in the kernel parameters.  Each thread reads its point once, walks the V views in
//              order in registers (the depth maps are gathered through L2) and stores only if a view updated it, so
//              unobserved space costs one read.  Per call: 8 B per point read (20 B with colour), as much written
//              where some view updated the point.
//   extract  : classify (per point: flags of its +x/+y/+z edges, its cell's validity and cube index, and per-block
//              vertex / face counts), block_sums_scan_kernel (scan.cuh, here over 64-bit sums) over those counts, one
//              copy of the totals to the host; then an emit pass for the vertices (block-local scan; it also stores
//              every point's first vertex index) and one for the faces (block-local scan; a face's indices are the
//              owner points' first vertex plus the edge's rank among the owner's flagged edges).  Vertex and face order
//              are the grid's, not the schedule's: the mesh is a function of the volume.
// No float atomics; all arithmetic is IEEE fp32 with correctly rounded division, so both parts are bitwise
// reproducible, and V views in one call give the bits of V one-view calls in the same order (the same operations on
// the same fp32 values, whether kept in registers or stored between calls).
#include <cmath>
#include "common.cuh"
#include "kernels.h"
#include "mc_table.cuh"
#include "scan.cuh"

namespace r3dg {
namespace {

constexpr int kIntThreads = 256;
constexpr int kExThreads = 256;
constexpr int kExItems = 4;                           // points per thread in the extraction passes
constexpr int kExTile = kExThreads * kExItems;        // points per block, item-major: base + it * kExThreads + tid

struct TsdfIntParams {
    int NX, NY, NZ, V, H, W;
    float ox, oy, oz, vs, sdf_trunc, depth_trunc;
    float fx[R3DG_MAX_VIEWS], fy[R3DG_MAX_VIEWS], cx[R3DG_MAX_VIEWS], cy[R3DG_MAX_VIEWS];
};

__global__ void __launch_bounds__(kIntThreads) tsdf_integrate_kernel(const TsdfIntParams p, float* __restrict__ tsdf,
                                                                    float* __restrict__ weight, float* __restrict__ color,
                                                                    const float* __restrict__ depth,
                                                                    const float* __restrict__ rgb,
                                                                    const float* __restrict__ viewmatrix) {
    __shared__ float s_view[R3DG_MAX_VIEWS * 16];
    for (int i = threadIdx.x; i < p.V * 16; i += blockDim.x) s_view[i] = viewmatrix[i];
    __syncthreads();
    const long long N = (long long)p.NX * p.NY * p.NZ;
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= N) return;
    const int k = (int)(g % p.NZ);
    const long long ij = g / p.NZ;
    const int j = (int)(ij % p.NY), i = (int)(ij / p.NY);
    const float x = p.ox + p.vs * (float)i, y = p.oy + p.vs * (float)j, z = p.oz + p.vs * (float)k;
    float t = tsdf[g], w = weight[g];
    float c0 = 0.f, c1 = 0.f, c2 = 0.f;
    if (color) { c0 = color[3 * g]; c1 = color[3 * g + 1]; c2 = color[3 * g + 2]; }
    const long long HW = (long long)p.H * p.W;
    bool updated = false;
    for (int v = 0; v < p.V; ++v) {
        const float* m = s_view + 16 * v;
        const float Z = x * m[2] + y * m[6] + z * m[10] + m[14];
        if (!(Z > 0.f)) continue;
        const float X = x * m[0] + y * m[4] + z * m[8] + m[12];
        const float Y = x * m[1] + y * m[5] + z * m[9] + m[13];
        const float pu = floorf(p.fx[v] * (X / Z) + p.cx[v] + 0.5f);
        const float pv = floorf(p.fy[v] * (Y / Z) + p.cy[v] + 0.5f);
        if (!(pu >= 0.f && pu < (float)p.W && pv >= 0.f && pv < (float)p.H)) continue;
        const long long pix = (long long)pv * p.W + (long long)pu;
        const float D = __ldg(depth + v * HW + pix);
        if (!(D > 0.f && D <= p.depth_trunc && isfinite(D))) continue;
        const float sdf = D - Z;
        if (!(sdf >= -p.sdf_trunc)) continue;
        const float obs = fminf(1.f, sdf / p.sdf_trunc);
        const float w1 = w + 1.f;
        t = (t * w + obs) / w1;
        if (color) {
            const float* im = rgb + 3 * v * HW + pix;
            c0 = (c0 * w + __ldg(im)) / w1;
            c1 = (c1 * w + __ldg(im + HW)) / w1;
            c2 = (c2 * w + __ldg(im + 2 * HW)) / w1;
        }
        w = w1;
        updated = true;
    }
    if (!updated) return;
    tsdf[g] = t;
    weight[g] = w;
    if (color) { color[3 * g] = c0; color[3 * g + 1] = c1; color[3 * g + 2] = c2; }
}

// Per-point code of the extraction: bits 0-2 the vertex flags of the point's +x/+y/+z edges, bit 3 the validity of the
// cell whose lower corner is the point, bits 8-15 that cell's cube index.
constexpr uint32_t kCellValid = 8u;

struct ExGrid {
    int NX, NY, NZ;
    long long N;
    float ox, oy, oz, vs;
};

__device__ __forceinline__ void point_ijk(const ExGrid& G, long long g, int& i, int& j, int& k) {
    k = (int)(g % G.NZ);
    const long long ij = g / G.NZ;
    j = (int)(ij % G.NY);
    i = (int)(ij / G.NY);
}

__device__ __forceinline__ int face_count(uint32_t code) { return (code & kCellValid) ? kMcCount[code >> 8] : 0; }

// exclusive prefix of v over the CTA's kExThreads threads, in thread order; *total = the CTA's sum.  Ends with a
// barrier, so s_warp can be reused by the next call.
__device__ __forceinline__ uint32_t cta_exclusive_scan(uint32_t v, uint32_t* s_warp, uint32_t* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    uint32_t before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < kExThreads / 32; ++w) {
        const uint32_t s = s_warp[w];
        before += w < warp ? s : 0u;
        all += s;
    }
    __syncthreads();
    *total = all;
    return before + inc - v;
}

__global__ void __launch_bounds__(kExThreads) tsdf_classify_kernel(const ExGrid G, const float* __restrict__ tsdf,
                                                                  const float* __restrict__ weight,
                                                                  uint16_t* __restrict__ code,
                                                                  unsigned long long* __restrict__ block_sums,
                                                                  long long nblocks) {
    __shared__ uint32_t s_v[kExThreads / 32], s_f[kExThreads / 32];
    const long long sy = G.NZ, sx = (long long)G.NY * G.NZ;
    uint32_t nv = 0, nf = 0;
    for (int it = 0; it < kExItems; ++it) {
        const long long g = (long long)blockIdx.x * kExTile + (long long)it * kExThreads + threadIdx.x;
        if (g >= G.N) break;
        int i, j, k;
        point_ijk(G, g, i, j, k);
        // observed (weight > 0) bits of the 3x3x3 neighbourhood, bit (di + 1) * 9 + (dj + 1) * 3 + (dk + 1)
        uint32_t obs = 0;
        for (int di = -1; di <= 1; ++di)
            for (int dj = -1; dj <= 1; ++dj)
                for (int dk = -1; dk <= 1; ++dk) {
                    const int a = i + di, b = j + dj, c = k + dk;
                    if (a < 0 || a >= G.NX || b < 0 || b >= G.NY || c < 0 || c >= G.NZ) continue;
                    if (weight[g + di * sx + dj * sy + dk] > 0.f) obs |= 1u << ((di + 1) * 9 + (dj + 1) * 3 + (dk + 1));
                }
        // validity of the 8 cells with lower corner (i + ci, j + cj, k + ck), ci, cj, ck in {-1, 0}: bit (ci+1)*4+(cj+1)*2+(ck+1)
        uint32_t cells = 0;
        for (int ci = -1; ci <= 0; ++ci)
            for (int cj = -1; cj <= 0; ++cj)
                for (int ck = -1; ck <= 0; ++ck) {
                    if (i + ci < 0 || i + ci + 1 >= G.NX || j + cj < 0 || j + cj + 1 >= G.NY || k + ck < 0 ||
                        k + ck + 1 >= G.NZ)
                        continue;
                    bool all = true;
                    for (int c = 0; c < 8; ++c)
                        all = all && ((obs >> ((ci + 1 + (c & 1)) * 9 + (cj + 1 + ((c >> 1) & 1)) * 3 +
                                               (ck + 1 + ((c >> 2) & 1)))) & 1u);
                    if (all) cells |= 1u << ((ci + 1) * 4 + (cj + 1) * 2 + (ck + 1));
                }
        // inside bits of the corners of the cell at (i, j, k) that exist
        uint32_t in = 0;
        for (int c = 0; c < 8; ++c) {
            const int di = c & 1, dj = (c >> 1) & 1, dk = (c >> 2) & 1;
            if (i + di >= G.NX || j + dj >= G.NY || k + dk >= G.NZ) continue;
            if (tsdf[g + di * sx + dj * sy + dk] < 0.f) in |= 1u << c;
        }
        uint32_t cd = 0;
        // +x edge: cells (i, j-1|j, k-1|k) = bits 4..7; +y: (i-1|i, j, k-1|k) = bits 2, 3, 6, 7; +z: bits 1, 3, 5, 7
        if (i + 1 < G.NX && ((in ^ (in >> 1)) & 1u) && (cells & 0xF0u)) cd |= 1u;
        if (j + 1 < G.NY && ((in ^ (in >> 2)) & 1u) && (cells & 0xCCu)) cd |= 2u;
        if (k + 1 < G.NZ && ((in ^ (in >> 4)) & 1u) && (cells & 0xAAu)) cd |= 4u;
        if (cells & 0x80u) cd |= kCellValid | (in << 8);
        code[g] = (uint16_t)cd;
        nv += __popc(cd & 7u);
        nf += face_count(cd);
    }
    nv = __reduce_add_sync(0xffffffffu, nv);
    nf = __reduce_add_sync(0xffffffffu, nf);
    if ((threadIdx.x & 31) == 0) { s_v[threadIdx.x >> 5] = nv; s_f[threadIdx.x >> 5] = nf; }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t a = 0, b = 0;
        for (int w = 0; w < kExThreads / 32; ++w) { a += s_v[w]; b += s_f[w]; }
        block_sums[blockIdx.x] = a;
        block_sums[nblocks + blockIdx.x] = b;
    }
}

__global__ void __launch_bounds__(kExThreads) tsdf_emit_verts_kernel(const ExGrid G, const float* __restrict__ tsdf,
                                                                    const float* __restrict__ color,
                                                                    const uint16_t* __restrict__ code,
                                                                    const unsigned long long* __restrict__ vert_base,
                                                                    uint32_t* __restrict__ first_vert,
                                                                    float* __restrict__ verts,
                                                                    float* __restrict__ vert_colors) {
    __shared__ uint32_t s_warp[kExThreads / 32];
    const long long step[3] = {(long long)G.NY * G.NZ, (long long)G.NZ, 1};
    uint32_t run = (uint32_t)vert_base[blockIdx.x];            // < 2^31: the count refused larger totals
    for (int it = 0; it < kExItems; ++it) {
        const long long g = (long long)blockIdx.x * kExTile + (long long)it * kExThreads + threadIdx.x;
        const uint32_t cd = g < G.N ? code[g] : 0u;
        uint32_t tot;
        uint32_t vid = run + cta_exclusive_scan(__popc(cd & 7u), s_warp, &tot);
        run += tot;
        if (g >= G.N) continue;
        first_vert[g] = vid;
        if (!(cd & 7u)) continue;
        int i, j, k;
        point_ijk(G, g, i, j, k);
        const float p0[3] = {G.ox + G.vs * (float)i, G.oy + G.vs * (float)j, G.oz + G.vs * (float)k};
        const float v0 = tsdf[g];
        for (int a = 0; a < 3; ++a) {
            if (!((cd >> a) & 1u)) continue;
            const long long g1 = g + step[a];
            const float v1 = tsdf[g1];
            const float t = v0 / (v0 - v1);
            float* out = verts + 3 * (long long)vid;
            out[0] = p0[0]; out[1] = p0[1]; out[2] = p0[2];
            out[a] = p0[a] + t * G.vs;
            if (color) {
                float* oc = vert_colors + 3 * (long long)vid;
                for (int c = 0; c < 3; ++c) {
                    const float a0 = color[3 * g + c], a1 = color[3 * g1 + c];
                    oc[c] = a0 + t * (a1 - a0);
                }
            }
            ++vid;
        }
    }
}

__global__ void __launch_bounds__(kExThreads) tsdf_emit_faces_kernel(const ExGrid G, const uint16_t* __restrict__ code,
                                                                    const unsigned long long* __restrict__ face_base,
                                                                    const uint32_t* __restrict__ first_vert,
                                                                    int* __restrict__ faces) {
    __shared__ uint32_t s_warp[kExThreads / 32];
    const long long sx = (long long)G.NY * G.NZ, sy = G.NZ;
    uint32_t run = (uint32_t)face_base[blockIdx.x];
    for (int it = 0; it < kExItems; ++it) {
        const long long g = (long long)blockIdx.x * kExTile + (long long)it * kExThreads + threadIdx.x;
        const uint32_t cd = g < G.N ? code[g] : 0u;
        const int nf = face_count(cd);
        uint32_t tot;
        const uint32_t fid = run + cta_exclusive_scan((uint32_t)nf, s_warp, &tot);
        run += tot;
        const uint32_t cube = cd >> 8;
        for (int s = 0; s < nf; ++s)
            for (int r = 0; r < 3; ++r) {
                const int e = kMcTris[cube][3 * s + r];
                const int a = kMcEdge[e][0], axis = e >> 2;
                const long long owner = g + (a & 1) * sx + ((a >> 1) & 1) * sy + ((a >> 2) & 1);
                const uint32_t oc = code[owner];
                faces[3 * ((long long)fid + s) + r] = (int)(first_vert[owner] + __popc(oc & 7u & ((1u << axis) - 1u)));
            }
    }
}

// work layout: u16 code [N], u32 first_vert [N], u64 block sums [2][nblocks], u64 totals [2]
struct ExLayout {
    size_t code, first_vert, sums, totals, total;
    long long nblocks;
    ExLayout(long long N) : nblocks((N + kExTile - 1) / kExTile) {
        size_t off = 0;
        code = off;       off = align_up(off + (size_t)N * 2, 256);
        first_vert = off; off = align_up(off + (size_t)N * 4, 256);
        sums = off;       off = align_up(off + (size_t)nblocks * 16, 256);
        totals = off;     off = align_up(off + 16, 256);
        total = off;
    }
};

bool finite_pos(float x) { return std::isfinite(x) && x > 0.f; }

// shared checks of the grid: R3DG_ERR_BAD_ARG / R3DG_ERR_UNSUPPORTED, 0 when fine
int check_grid(int NX, int NY, int NZ, const float* origin, float voxel_size) {
    if (NX < 2 || NY < 2 || NZ < 2) return R3DG_ERR_BAD_ARG;
    if (!std::isfinite(origin[0]) || !std::isfinite(origin[1]) || !std::isfinite(origin[2]) || !finite_pos(voxel_size))
        return R3DG_ERR_BAD_ARG;
    if ((long long)NX * NY * NZ >= (1LL << 31)) return R3DG_ERR_UNSUPPORTED;
    return 0;
}

ExGrid ex_grid(const r3dg_tsdf_extract_args* a) {
    ExGrid G;
    G.NX = a->NX; G.NY = a->NY; G.NZ = a->NZ;
    G.N = (long long)a->NX * a->NY * a->NZ;
    G.ox = a->origin[0]; G.oy = a->origin[1]; G.oz = a->origin[2]; G.vs = a->voxel_size;
    return G;
}

}  // namespace

size_t tsdf_extract_work_bytes(int NX, int NY, int NZ) {
    const long long N = (long long)(NX < 2 ? 2 : NX) * (NY < 2 ? 2 : NY) * (NZ < 2 ? 2 : NZ);
    return ExLayout(N).total;
}

int launch_tsdf_integrate(const r3dg_tsdf_integrate_args* a, cudaStream_t stream) {
    if (!a) return R3DG_ERR_BAD_ARG;
    int rc = check_grid(a->NX, a->NY, a->NZ, a->origin, a->voxel_size);
    if (rc == R3DG_ERR_BAD_ARG) return rc;
    if (!finite_pos(a->sdf_trunc) || !(a->depth_trunc > 0.f)) return R3DG_ERR_BAD_ARG;
    if (a->V < 1 || a->V > R3DG_MAX_VIEWS || a->H < 1 || a->W < 1) return R3DG_ERR_BAD_ARG;
    if (!a->tsdf || !a->weight || !a->depth || !a->viewmatrix || !a->cams) return R3DG_ERR_BAD_ARG;
    if ((a->color == nullptr) != (a->rgb == nullptr)) return R3DG_ERR_BAD_ARG;
    TsdfIntParams p;
    for (int v = 0; v < a->V; ++v) {
        const float* c = a->cams + 4 * v;
        if (!finite_pos(c[0]) || !finite_pos(c[1]) || !std::isfinite(c[2]) || !std::isfinite(c[3])) return R3DG_ERR_BAD_ARG;
        p.fx[v] = (float)(a->W / (2.0 * c[0]));
        p.fy[v] = (float)(a->H / (2.0 * c[1]));
        p.cx[v] = c[2];
        p.cy[v] = c[3];
        if (!std::isfinite(p.fx[v]) || !std::isfinite(p.fy[v])) return R3DG_ERR_BAD_ARG;
    }
    if (rc != 0) return rc;
    if ((long long)a->H * a->W >= (1LL << 31)) return R3DG_ERR_UNSUPPORTED;
    p.NX = a->NX; p.NY = a->NY; p.NZ = a->NZ; p.V = a->V; p.H = a->H; p.W = a->W;
    p.ox = a->origin[0]; p.oy = a->origin[1]; p.oz = a->origin[2];
    p.vs = a->voxel_size; p.sdf_trunc = a->sdf_trunc; p.depth_trunc = a->depth_trunc;
    const long long N = (long long)a->NX * a->NY * a->NZ;
    tsdf_integrate_kernel<<<(unsigned)((N + kIntThreads - 1) / kIntThreads), kIntThreads, 0, stream>>>(
        p, a->tsdf, a->weight, a->color, a->depth, a->rgb, a->viewmatrix);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_tsdf_extract_count(const r3dg_tsdf_extract_args* a, cudaStream_t stream, bool* launched) {
    *launched = false;
    if (!a) return R3DG_ERR_BAD_ARG;
    const int rc = check_grid(a->NX, a->NY, a->NZ, a->origin, a->voxel_size);
    if (rc != 0) return rc;
    if (!a->tsdf || !a->weight || !a->work || !a->totals_host) return R3DG_ERR_BAD_ARG;
    const ExGrid G = ex_grid(a);
    const ExLayout L(G.N);
    if (a->work_bytes < L.total) return R3DG_ERR_BAD_ARG;
    char* w = (char*)a->work;
    unsigned long long* sums = (unsigned long long*)(w + L.sums);
    unsigned long long* totals = (unsigned long long*)(w + L.totals);
    tsdf_classify_kernel<<<(unsigned)L.nblocks, kExThreads, 0, stream>>>(G, a->tsdf, a->weight, (uint16_t*)(w + L.code),
                                                                         sums, L.nblocks);
    R3DG_CUDA_TRY(cudaGetLastError());
    block_sums_scan_kernel<2, unsigned long long><<<1, 1024, 0, stream>>>(L.nblocks, L.nblocks, sums, totals);
    R3DG_CUDA_TRY(cudaGetLastError());
    *launched = true;
    unsigned long long t[2];
    R3DG_CUDA_TRY(cudaMemcpyAsync(t, totals, sizeof(t), cudaMemcpyDeviceToHost, stream));
    R3DG_CUDA_TRY(cudaStreamSynchronize(stream));
    a->totals_host[0] = (long long)t[0];
    a->totals_host[1] = (long long)t[1];
    if (t[0] >= (1ULL << 31) || t[1] >= (1ULL << 31)) return R3DG_ERR_UNSUPPORTED;
    return 0;
}

int launch_tsdf_extract_emit(const r3dg_tsdf_extract_args* a, cudaStream_t stream) {
    if (!a) return R3DG_ERR_BAD_ARG;
    const int rc = check_grid(a->NX, a->NY, a->NZ, a->origin, a->voxel_size);
    if (rc != 0) return rc;
    if (!a->tsdf || !a->weight || !a->work) return R3DG_ERR_BAD_ARG;
    if (a->n_verts < 0 || a->n_faces < 0 || a->n_verts >= (1LL << 31) || a->n_faces >= (1LL << 31)) return R3DG_ERR_BAD_ARG;
    if ((a->n_verts > 0 && (!a->verts || (a->color && !a->vert_colors))) || (a->n_faces > 0 && !a->faces))
        return R3DG_ERR_BAD_ARG;
    const ExGrid G = ex_grid(a);
    const ExLayout L(G.N);
    if (a->work_bytes < L.total) return R3DG_ERR_BAD_ARG;
    if (a->n_verts == 0 && a->n_faces == 0) return 0;
    char* w = (char*)a->work;
    const uint16_t* code = (const uint16_t*)(w + L.code);
    uint32_t* first_vert = (uint32_t*)(w + L.first_vert);
    const unsigned long long* sums = (const unsigned long long*)(w + L.sums);
    tsdf_emit_verts_kernel<<<(unsigned)L.nblocks, kExThreads, 0, stream>>>(G, a->tsdf, a->color, code, sums, first_vert,
                                                                           a->verts, a->vert_colors);
    R3DG_CUDA_TRY(cudaGetLastError());
    tsdf_emit_faces_kernel<<<(unsigned)L.nblocks, kExThreads, 0, stream>>>(G, code, sums + L.nblocks, first_vert, a->faces);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace r3dg
