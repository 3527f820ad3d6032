// render_mesh.cu -- the mesh renderer behind the C ABI (include/uhc_render.h uhc_render_mesh_init / uhc_render_mesh):
//   k_mesh_refit        one block per (frame, humanoid): the box of every leaf's vertices, then every body's box as the union of its leaves'
//   k_render_mesh_trace 16 x 16 pixel tiles, blockIdx.z = frame: the frame's body and leaf boxes and the topology's ranges staged in shared
//                       memory, then per pixel render_core.h's shade_pixel over the mesh (render_mesh_core.h): floor, body boxes, leaf boxes,
//                       watertight ray-triangle tests, one shadow ray
//
// Compiled on its own with -fmad=false (uhc_b200/build.py): the pixel path must give the host emulation's bits.
#include <cuda_runtime.h>
#include <math.h>
#include <string>
#include "../../include/uhc_render.h"
#include "engine_slots.h"
#include "errors.h"
#define UHC_RENDER_HOST 1
#include "render_mesh_core.h"

using namespace uhc;

namespace {

constexpr int TILE = 16, SLOTS = 2 * render::NB, REFIT_THREADS = 128;
constexpr size_t SMEM_MAX = 200 * 1024;

struct MeshCtx {
    int nvert = 0, nface = 0, nleaf = 0;
    int *d_face = nullptr, *d_leaf_first = nullptr, *d_body_leaf = nullptr;
    float *d_box = nullptr; size_t box_cap = 0;        // refitted boxes, frames: [n][SLOTS + 2 nleaf][6]
};
MeshCtx *find_ctx(const UhcEngine *e) { return (MeshCtx *)engine_slot(e, SLOT_RENDER_MESH); }

__host__ __device__ size_t frame_boxes(int nleaf) { return (size_t)(SLOTS + 2 * nleaf) * 6; }     // floats per frame
size_t trace_smem(int nleaf) { return frame_boxes(nleaf) * sizeof(float) + (size_t)(nleaf + 1 + render::NB + 1) * sizeof(int); }

__global__ void __launch_bounds__(REFIT_THREADS) k_mesh_refit(long n, int nh, int nvert, int nleaf, const float *__restrict__ verts,
                                                               const float *__restrict__ ghost, float shift, const int *__restrict__ face,
                                                               const int *__restrict__ leaf_first, const int *__restrict__ body_leaf,
                                                               float *__restrict__ box) {
    const long i = blockIdx.x;                       // (frame, humanoid)
    const long f = i / nh;
    const int h = (int)(i - f * nh);
    const float *v = (h ? ghost : verts) + (size_t)f * nvert * 3;
    float *fb = box + (size_t)f * frame_boxes(nleaf);
    float *leaf = fb + SLOTS * 6 + (size_t)h * nleaf * 6;
    for (int l = threadIdx.x; l < nleaf; l += REFIT_THREADS) render::refit_leaf(v, face, leaf_first[l], leaf_first[l + 1], h, shift, leaf + 6 * l);
    __syncthreads();                                 // the block's leaf boxes are written (and visible to the block)
    if (threadIdx.x < render::NB) {
        const int b = threadIdx.x;
        render::union_boxes(leaf, body_leaf[b], body_leaf[b + 1], fb + 6 * (h * render::NB + b));
    }
}

struct MeshTraceArgs {
    render::Cam cam;
    int W, H, nh, nleaf, nvert;
    long n;
    const float *verts, *ghost, *root, *box;
    const int *face, *leaf_first, *body_leaf;
    unsigned char *rgb, *label;
    float *depth;
};

__global__ void __launch_bounds__(TILE * TILE) k_render_mesh_trace(const __grid_constant__ MeshTraceArgs a) {
    extern __shared__ float shm[];
    float *s_box = shm;                                             // [SLOTS][6] body boxes, then [2][nleaf][6] leaf boxes
    int *s_leaf_first = (int *)(shm + frame_boxes(a.nleaf));        // [nleaf + 1]
    int *s_body_leaf = s_leaf_first + a.nleaf + 1;                  // [25]
    const int tid = threadIdx.y * TILE + threadIdx.x;
    for (int k = tid; k <= a.nleaf; k += TILE * TILE) s_leaf_first[k] = a.leaf_first[k];
    if (tid <= render::NB) s_body_leaf[tid] = a.body_leaf[tid];
    const int x = blockIdx.x * TILE + threadIdx.x, y = blockIdx.y * TILE + threadIdx.y;
    const int nbody = a.nh * render::NB * 6, nleafbox = a.nh * a.nleaf * 6;
    for (long f = blockIdx.z; f < a.n; f += gridDim.z) {
        const float *fb = a.box + (size_t)f * frame_boxes(a.nleaf);
        __syncthreads();                                            // the previous frame's pixels are done with the staging
        for (int k = tid; k < nbody; k += TILE * TILE) s_box[k] = fb[k];
        for (int k = tid; k < nleafbox; k += TILE * TILE) s_box[SLOTS * 6 + k] = fb[SLOTS * 6 + k];
        __syncthreads();
        if (x >= a.W || y >= a.H) continue;
        render::MeshScene s;
        s.verts[0] = a.verts + (size_t)f * a.nvert * 3;
        s.verts[1] = a.ghost ? a.ghost + (size_t)f * a.nvert * 3 : s.verts[0];
        s.face = a.face; s.leaf_first = s_leaf_first; s.body_leaf = s_body_leaf;
        s.body_box = s_box; s.leaf_box = s_box + SLOTS * 6;
        s.nleaf = a.nleaf; s.visible = a.cam.visible; s.shift = a.cam.shift;
        s.root = a.root ? a.root + 3 * (size_t)f : nullptr;
        const size_t px = ((size_t)f * a.H + y) * a.W + x;
        unsigned char rgb[3], lab;
        float dep;
        render::shade_pixel(a.cam, s, x, y, a.W, a.H, rgb, &dep, &lab);
        a.rgb[3 * px] = rgb[0]; a.rgb[3 * px + 1] = rgb[1]; a.rgb[3 * px + 2] = rgb[2];
        if (a.depth) a.depth[px] = dep;
        if (a.label) a.label[px] = lab;
    }
}

}  // namespace

namespace uhc {
void render_mesh_release(UhcEngine *e) {
    MeshCtx *c = e ? find_ctx(e) : nullptr;
    if (!c) return;
    cudaFree(c->d_face); cudaFree(c->d_leaf_first); cudaFree(c->d_body_leaf); cudaFree(c->d_box);
    delete c; engine_slot(e, SLOT_RENDER_MESH) = nullptr;
}
}  // namespace uhc

extern "C" {

int uhc_render_mesh_init(UhcEngine *e, const UhcRenderMesh *m) {
    if (!e || !m) { uhc_err() = "uhc_render_mesh_init: null argument"; return -2; }
    const char *why = nullptr;
    if (render::mesh_tables_check(*m, &why)) { uhc_err() = std::string("uhc_render_mesh_init: ") + why; return -2; }
    if (trace_smem(m->nleaf) > SMEM_MAX) { uhc_err() = "uhc_render_mesh_init: the leaf boxes of two humanoids do not fit the trace's shared memory"; return -2; }
    uhc::render_mesh_release(e);
    MeshCtx *c = new MeshCtx();
    engine_slot(e, SLOT_RENDER_MESH) = c;
    c->nvert = m->nvert; c->nface = m->nface; c->nleaf = m->nleaf;
    CK(cudaMalloc((void **)&c->d_face, (size_t)m->nface * 3 * sizeof(int)));
    CK(cudaMalloc((void **)&c->d_leaf_first, (size_t)(m->nleaf + 1) * sizeof(int)));
    CK(cudaMalloc((void **)&c->d_body_leaf, (size_t)(render::NB + 1) * sizeof(int)));
    CK(cudaMemcpy(c->d_face, m->face, (size_t)m->nface * 3 * sizeof(int), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(c->d_leaf_first, m->leaf_first, (size_t)(m->nleaf + 1) * sizeof(int), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(c->d_body_leaf, m->body_leaf, (size_t)(render::NB + 1) * sizeof(int), cudaMemcpyHostToDevice));
    // the init's limit, not this model's need: the attribute is per function, and a smaller model on another engine must not lower it
    CK(cudaFuncSetAttribute(k_render_mesh_trace, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_MAX));
    CK(cudaDeviceSynchronize());
    return 0;
}

int uhc_render_mesh(UhcEngine *e, const UhcRenderCamera *cam, int W, int H, long n, const float *verts_dev, const float *ghost_verts_dev_or_null,
                    const float *root_dev_or_null, int nvert, unsigned char *rgb_dev, float *depth_dev_or_null, unsigned char *label_dev_or_null,
                    void *stream) {
    const char *who = "uhc_render_mesh: ";
    if (!e) { uhc_err() = std::string(who) + "null engine"; return -2; }
    MeshCtx *c = find_ctx(e);
    if (!c) { uhc_err() = std::string(who) + "no mesh tables (uhc_render_mesh_init)"; return -2; }
    if (const char *why = render::frame_args_error(cam, W, H, n)) { uhc_err() = std::string(who) + why; return -2; }
    if (nvert != c->nvert) { uhc_err() = std::string(who) + "nvert differs from uhc_render_mesh_init's"; return -2; }
    if (n > 0 && (!verts_dev || !rgb_dev)) { uhc_err() = std::string(who) + "null verts or rgb"; return -2; }
    if (n > 0 && cam->focus && !root_dev_or_null) { uhc_err() = std::string(who) + "a camera with focus needs the root"; return -2; }
    if (n == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    const int nh = ghost_verts_dev_or_null ? 2 : 1;
    if ((size_t)n > c->box_cap) {
        CK(cudaStreamSynchronize(st));                             // an earlier call on this stream may still read the old boxes
        cudaFree(c->d_box); c->d_box = nullptr; c->box_cap = 0;
        CK(cudaMalloc((void **)&c->d_box, (size_t)n * frame_boxes(c->nleaf) * sizeof(float)));
        c->box_cap = (size_t)n;
    }
    MeshTraceArgs a;
    render::camera_setup(*cam, W, H, nh, &a.cam);
    k_mesh_refit<<<(unsigned)(n * nh), REFIT_THREADS, 0, st>>>(n, nh, nvert, c->nleaf, verts_dev, ghost_verts_dev_or_null, a.cam.shift, c->d_face,
                                                               c->d_leaf_first, c->d_body_leaf, c->d_box);
    CK(cudaGetLastError());
    a.W = W; a.H = H; a.nh = nh; a.nleaf = c->nleaf; a.nvert = nvert; a.n = n;
    a.verts = verts_dev; a.ghost = ghost_verts_dev_or_null; a.root = root_dev_or_null; a.box = c->d_box;
    a.face = c->d_face; a.leaf_first = c->d_leaf_first; a.body_leaf = c->d_body_leaf;
    a.rgb = rgb_dev; a.depth = depth_dev_or_null; a.label = label_dev_or_null;
    const dim3 grid((unsigned)((W + TILE - 1) / TILE), (unsigned)((H + TILE - 1) / TILE), (unsigned)(n < 65535 ? n : 65535));
    k_render_mesh_trace<<<grid, dim3(TILE, TILE), trace_smem(c->nleaf), st>>>(a);
    CK(cudaGetLastError());
    return 0;
}

}  // extern "C"
