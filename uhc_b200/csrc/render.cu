// render.cu -- the offline renderer behind the C ABI (include/uhc_render.h):
//   k_render_pose   one thread per (frame, humanoid): qpos -> fp64 FK (motion_core.h) with the frame's shape variant -> fp32 pose rows
//   k_render_trace  16 x 16 pixel tiles, blockIdx.z = frame: the variant's hull planes and the frame's poses / world spheres staged in shared
//                   memory, then per pixel one primary ray (floor z = 0 and every hull, Cyrus-Beck) and one shadow ray (render_core.h)
//
// Compiled on its own with -fmad=false (uhc_b200/build.py): render_core.h's fp32 pixel path must give the host emulation's bits.
#include <cuda_runtime.h>
#include <math.h>
#include <string>
#include <vector>
#include "../../include/uhc_render.h"
#include "engine_slots.h"
#include "errors.h"
#define UHC_RENDER_HOST 1
#include "render_core.h"
#include "track_glue.h"

using namespace uhc;

namespace uhc { void render_mesh_release(UhcEngine *e); }   // render_mesh.cu: the mesh tables and their scratch

namespace {

constexpr int TILE = 16, SLOTS = 2 * render::NB;
constexpr size_t SMEM_MAX = 200 * 1024;                // dynamic shared memory of a trace, at most

struct RenderCtx {
    int nshape = 0, nplane = 0;
    int adr[render::NB], num[render::NB];
    float4 *d_plane = nullptr, *d_sphere = nullptr;    // [nshape][nplane], [nshape][24]
    float *d_pose = nullptr; size_t pose_cap = 0;      // uhc_render_qpos' pose table, frames
};
RenderCtx *find_ctx(const UhcEngine *e) { return (RenderCtx *)engine_slot(e, SLOT_RENDER); }
void free_ctx(UhcEngine *e) {
    RenderCtx *c = find_ctx(e);
    if (!c) return;
    cudaFree(c->d_plane); cudaFree(c->d_sphere); cudaFree(c->d_pose);
    delete c; engine_slot(e, SLOT_RENDER) = nullptr;
}

template <class Real>
__global__ void __launch_bounds__(128) k_render_pose(motion::MotionModel m, long n, int nh, const Real *__restrict__ q0, long pitch0,
                                                     const Real *__restrict__ q1, long pitch1, const int *__restrict__ variant, float *__restrict__ pose) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * nh) return;
    const long f = i / nh;
    const int h = (int)(i - f * nh);
    const Real *src = h == 0 ? q0 + (size_t)f * pitch0 : q1 + (size_t)f * pitch1;
    double q[motion::MQ], wpos[3 * motion::MB], wq[4 * motion::MB];
    for (int k = 0; k < motion::MQ; k++) q[k] = (double)src[k];
    render::pose_fk(m, q, m.body + (size_t)(variant ? variant[f] : 0) * motion::MB * motion::BODY6, wpos, wq);
    render::pose_rows<float>(wpos, wq, pose + ((size_t)f * 2 + h) * render::NB * render::POSE);
}

struct TraceArgs {
    render::Cam cam;
    int W, H, nh, nplane;
    long n;
    const float *pose;
    const int *variant;
    const float4 *plane, *sphere;
    int adr[render::NB], num[render::NB];
    unsigned char *rgb, *label;
    float *depth;
};

__global__ void __launch_bounds__(TILE * TILE) k_render_trace(const __grid_constant__ TraceArgs a) {
    extern __shared__ float4 sh[];
    float4 *s_plane = sh;                                           // [nplane]
    float *s_pose = (float *)(sh + a.nplane);                       // [48][POSE]
    float *s_sph = s_pose + SLOTS * render::POSE;                   // [48][4]
    __shared__ int s_adr[render::NB], s_num[render::NB];
    const int tid = threadIdx.y * TILE + threadIdx.x;
    if (tid < render::NB) { s_adr[tid] = a.adr[tid]; s_num[tid] = a.num[tid]; }
    const int x = blockIdx.x * TILE + threadIdx.x, y = blockIdx.y * TILE + threadIdx.y;
    for (long f = blockIdx.z; f < a.n; f += gridDim.z) {
        const float4 *pl = a.plane + (size_t)(a.variant ? a.variant[f] : 0) * a.nplane;
        const float4 *sp = a.sphere + (size_t)(a.variant ? a.variant[f] : 0) * render::NB;
        __syncthreads();                                            // the previous frame's pixels are done with the staging
        for (int k = tid; k < a.nplane; k += TILE * TILE) s_plane[k] = pl[k];
        if (tid < render::NB * a.nh) {
            const int h = tid / render::NB, b = tid - h * render::NB;
            const float4 c = sp[b];
            const float cs[4] = {c.x, c.y, c.z, c.w};
            render::stage_body(a.pose + ((size_t)f * 2 + h) * render::NB * render::POSE + b * render::POSE, cs, h, a.cam.shift,
                               s_pose + tid * render::POSE, s_sph + 4 * tid);
        }
        __syncthreads();
        if (x >= a.W || y >= a.H) continue;
        render::Scene s;
        s.plane = (const float *)s_plane; s.adr = s_adr; s.num = s_num; s.pose = s_pose; s.sph = s_sph; s.visible = a.cam.visible;
        const size_t px = ((size_t)f * a.H + y) * a.W + x;
        unsigned char rgb[3], lab;
        float dep;
        render::shade_pixel(a.cam, s, x, y, a.W, a.H, rgb, &dep, &lab);
        a.rgb[3 * px] = rgb[0]; a.rgb[3 * px + 1] = rgb[1]; a.rgb[3 * px + 2] = rgb[2];
        if (a.depth) a.depth[px] = dep;
        if (a.label) a.label[px] = lab;
    }
}

size_t trace_smem(int nplane) { return (size_t)nplane * sizeof(float4) + (size_t)SLOTS * (render::POSE + 4) * sizeof(float); }

// the variant array on the host, range-checked (-2), or -1 on a CUDA error
int check_variants(UhcEngine *e, long n, const int *variant_dev, cudaStream_t st, const char *who) {
    if (!variant_dev || n == 0) return 0;
    std::vector<int> v((size_t)n);
    CK(cudaMemcpyAsync(v.data(), variant_dev, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    const int ns = trackx::num_shapes(e);
    for (long i = 0; i < n; i++)
        if (v[(size_t)i] < 0 || v[(size_t)i] >= ns) { uhc_err() = std::string(who) + ": variant out of range"; return -2; }
    return 0;
}

int pose_args(UhcEngine *e, long n, const void *qpos, int precision, long pitch, const void *ghost, long ghost_pitch, const char *who) {
    if (!e) { uhc_err() = std::string(who) + ": null engine"; return -2; }
    if (n < 0) { uhc_err() = std::string(who) + ": n < 0"; return -2; }
    if (precision != 32 && precision != 64) { uhc_err() = std::string(who) + ": precision must be 32 or 64"; return -2; }
    if (pitch < motion::MQ || (ghost && ghost_pitch < motion::MQ)) { uhc_err() = std::string(who) + ": pitch < 76"; return -2; }
    if (n > 0 && !qpos) { uhc_err() = std::string(who) + ": null qpos"; return -2; }
    return 0;
}

int launch_pose(UhcEngine *e, long n, const void *qpos, int precision, long pitch, const void *ghost, long ghost_pitch, const int *variant,
                float *pose, cudaStream_t st) {
    if (n == 0) return 0;
    const int nh = ghost ? 2 : 1;
    const long threads = n * nh;
    const unsigned blocks = (unsigned)((threads + 127) / 128);
    const motion::MotionModel &m = trackx::motion_model(e);
    if (precision == 32)
        k_render_pose<float><<<blocks, 128, 0, st>>>(m, n, nh, (const float *)qpos, pitch, (const float *)ghost, ghost_pitch, variant, pose);
    else
        k_render_pose<double><<<blocks, 128, 0, st>>>(m, n, nh, (const double *)qpos, pitch, (const double *)ghost, ghost_pitch, variant, pose);
    CK(cudaGetLastError());
    return 0;
}

// argument checks of a trace (-2 with nothing launched)
int trace_args(UhcEngine *e, const UhcRenderCamera *cam, int W, int H, long n, int humanoids, const void *pose, const void *rgb, const char *who) {
    if (!e) { uhc_err() = std::string(who) + ": null engine"; return -2; }
    if (!find_ctx(e)) { uhc_err() = std::string(who) + ": no hull planes (uhc_render_init)"; return -2; }
    if (const char *why = render::frame_args_error(cam, W, H, n)) { uhc_err() = std::string(who) + ": " + why; return -2; }
    if (humanoids != 1 && humanoids != 2) { uhc_err() = std::string(who) + ": humanoids must be 1 or 2"; return -2; }
    if (n > 0 && (!pose || !rgb)) { uhc_err() = std::string(who) + ": null pose or rgb"; return -2; }
    return 0;
}

int launch_trace(RenderCtx *c, const UhcRenderCamera *cam, int W, int H, long n, const float *pose, int nh, const int *variant, unsigned char *rgb,
                 float *depth, unsigned char *label, cudaStream_t st) {
    if (n == 0) return 0;
    TraceArgs a;
    render::camera_setup(*cam, W, H, nh, &a.cam);
    a.W = W; a.H = H; a.nh = nh; a.nplane = c->nplane; a.n = n; a.pose = pose; a.variant = variant;
    a.plane = c->d_plane; a.sphere = c->d_sphere;
    for (int b = 0; b < render::NB; b++) { a.adr[b] = c->adr[b]; a.num[b] = c->num[b]; }
    a.rgb = rgb; a.depth = depth; a.label = label;
    const dim3 grid((unsigned)((W + TILE - 1) / TILE), (unsigned)((H + TILE - 1) / TILE), (unsigned)(n < 65535 ? n : 65535));
    k_render_trace<<<grid, dim3(TILE, TILE), trace_smem(c->nplane), st>>>(a);
    CK(cudaGetLastError());
    return 0;
}

}  // namespace

extern "C" {

int uhc_render_init(UhcEngine *e, const UhcRenderHulls *h) {
    if (!e || !h || !h->plane || !h->plane_adr || !h->plane_num || !h->sphere) { uhc_err() = "uhc_render_init: null argument"; return -2; }
    if (h->nshape != trackx::num_shapes(e)) { uhc_err() = "uhc_render_init: nshape differs from the engine's shape variants"; return -2; }
    if (h->nplane < 4 || trace_smem(h->nplane) > SMEM_MAX) { uhc_err() = "uhc_render_init: nplane out of range"; return -2; }
    for (int b = 0; b < render::NB; b++)
        if (h->plane_num[b] < 4 || h->plane_num[b] > UHC_RENDER_MAX_PLANES || h->plane_adr[b] < 0 || h->plane_adr[b] > h->nplane - h->plane_num[b]) {
            uhc_err() = "uhc_render_init: plane_adr / plane_num of a body out of range"; return -2;
        }
    const size_t np = (size_t)h->nshape * h->nplane, ns = (size_t)h->nshape * render::NB;
    std::vector<float4> pl(np), sp(ns);
    for (size_t i = 0; i < np; i++) {
        const double *p = h->plane + 4 * i;
        if (!(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]) && isfinite(p[3]))) { uhc_err() = "uhc_render_init: non-finite plane"; return -2; }
        pl[i] = make_float4((float)p[0], (float)p[1], (float)p[2], (float)p[3]);
    }
    for (size_t i = 0; i < ns; i++) {
        const double *p = h->sphere + 4 * i;
        if (!(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]) && p[3] > 0 && isfinite(p[3]))) { uhc_err() = "uhc_render_init: bad bounding sphere"; return -2; }
        sp[i] = make_float4((float)p[0], (float)p[1], (float)p[2], (float)p[3]);
    }
    free_ctx(e);                                                  // the mesh tables (uhc_render_mesh_init) stay
    RenderCtx *c = new RenderCtx();
    engine_slot(e, SLOT_RENDER) = c;
    c->nshape = h->nshape; c->nplane = h->nplane;
    for (int b = 0; b < render::NB; b++) { c->adr[b] = h->plane_adr[b]; c->num[b] = h->plane_num[b]; }
    CK(cudaMalloc((void **)&c->d_plane, np * sizeof(float4)));
    CK(cudaMalloc((void **)&c->d_sphere, ns * sizeof(float4)));
    CK(cudaMemcpy(c->d_plane, pl.data(), np * sizeof(float4), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(c->d_sphere, sp.data(), ns * sizeof(float4), cudaMemcpyHostToDevice));
    // the init's limit, not these planes' need: the attribute is per function, and fewer planes on another engine must not lower it
    CK(cudaFuncSetAttribute(k_render_trace, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_MAX));
    CK(cudaDeviceSynchronize());
    return 0;
}

void uhc_render_release(UhcEngine *e) {
    if (!e) return;
    free_ctx(e);
    uhc::render_mesh_release(e);
}

int uhc_render_pose(UhcEngine *e, long n, const void *qpos_dev, int precision, long pitch, const void *ghost_qpos_dev_or_null, long ghost_pitch,
                    const int *variant_dev_or_null, float *pose_dev, void *stream) {
    if (int rc = pose_args(e, n, qpos_dev, precision, pitch, ghost_qpos_dev_or_null, ghost_pitch, "uhc_render_pose")) return rc;
    if (n > 0 && !pose_dev) { uhc_err() = "uhc_render_pose: null pose"; return -2; }
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = check_variants(e, n, variant_dev_or_null, st, "uhc_render_pose")) return rc;
    return launch_pose(e, n, qpos_dev, precision, pitch, ghost_qpos_dev_or_null, ghost_pitch, variant_dev_or_null, pose_dev, st);
}

int uhc_render_bodies(UhcEngine *e, const UhcRenderCamera *cam, int W, int H, long n, const float *pose_dev, int humanoids,
                      const int *variant_dev_or_null, unsigned char *rgb_dev, float *depth_dev_or_null, unsigned char *label_dev_or_null, void *stream) {
    if (int rc = trace_args(e, cam, W, H, n, humanoids, pose_dev, rgb_dev, "uhc_render_bodies")) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = check_variants(e, n, variant_dev_or_null, st, "uhc_render_bodies")) return rc;
    return launch_trace(find_ctx(e), cam, W, H, n, pose_dev, humanoids, variant_dev_or_null, rgb_dev, depth_dev_or_null, label_dev_or_null, st);
}

int uhc_render_qpos(UhcEngine *e, const UhcRenderCamera *cam, int W, int H, long n, const void *qpos_dev, int precision, long pitch,
                    const void *ghost_qpos_dev_or_null, long ghost_pitch, const int *variant_dev_or_null, unsigned char *rgb_dev,
                    float *depth_dev_or_null, unsigned char *label_dev_or_null, void *stream) {
    const int nh = ghost_qpos_dev_or_null ? 2 : 1;
    if (int rc = trace_args(e, cam, W, H, n, nh, n > 0 ? (const void *)qpos_dev : nullptr, rgb_dev, "uhc_render_qpos")) return rc;
    if (int rc = pose_args(e, n, qpos_dev, precision, pitch, ghost_qpos_dev_or_null, ghost_pitch, "uhc_render_qpos")) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = check_variants(e, n, variant_dev_or_null, st, "uhc_render_qpos")) return rc;
    if (n == 0) return 0;
    RenderCtx *c = find_ctx(e);
    if ((size_t)n > c->pose_cap) {
        CK(cudaStreamSynchronize(st));                             // an earlier call on this stream may still read the old table
        cudaFree(c->d_pose); c->d_pose = nullptr; c->pose_cap = 0;
        CK(cudaMalloc((void **)&c->d_pose, (size_t)n * SLOTS * render::POSE * sizeof(float)));
        c->pose_cap = (size_t)n;
    }
    if (int rc = launch_pose(e, n, qpos_dev, precision, pitch, ghost_qpos_dev_or_null, ghost_pitch, variant_dev_or_null, c->d_pose, st)) return rc;
    return launch_trace(c, cam, W, H, n, c->d_pose, nh, variant_dev_or_null, rgb_dev, depth_dev_or_null, label_dev_or_null, st);
}

}  // extern "C"
