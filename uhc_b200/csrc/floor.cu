// floor.cu -- the body hulls against the floor behind the C ABI (include/uhc_floor.h), one warp per frame (floor_core.h):
//   k_floor_qpos    frames of a qpos array at any pitch (plain qpos, the evaluation's state record, the tracker's state_out)
//   k_floor_motion  frames of raw SMPL / qpos rows, converted by the code of uhc_load_motions (motion_core.h m_load_qpos)
//   k_eval_floor    the evaluation's recorded frame of every env, inside its graph (eval.cu)
// Lanes 0 and 1 place the bodies of the frame and of its previous frame (the renderer's fp64 pose pass), then all lanes take the hull
// vertices strided in vertex order and merge their partial results in a fixed butterfly.
//
// Compiled on its own with -fmad=false (uhc_b200/build.py) like motion_lib.cu and export.cu: floor_core.h must give the bits of its host
// emulation wherever the math library does.  sm_90a.
#include <cuda_runtime.h>
#include <string.h>
#include <string>
#include <vector>
#include "../../include/uhc_floor.h"
#include "../../include/uhc_track.h"
#include "errors.h"
#include "eval_glue.h"
#include "floor_core.h"
#include "sim_core.h"
#include "track_glue.h"

using namespace uhc;

namespace {

constexpr int WARPS = 4;   // frames per block
constexpr unsigned FULL = 0xffffffffu;

// vert = [nshape][nvert][3]; variant nshape + env is env's run-time subject (uhc_track_set_subjects), whose vertices are slot [env][nvert][3]
struct FloorDev { const double *vert; const unsigned char *vbody; int nvert, nshape; const double *slot; };

struct FloorCtx {
    UhcEngine *eng = nullptr;
    int nshape = 0;
    unsigned long long gen = 0;        // of this upload: graphs that hold `dev` carry it in their key
    double *d_vert = nullptr; unsigned char *d_vbody = nullptr;
    FloorDev dev{};
};
std::vector<FloorCtx *> g_fl;
unsigned long long g_fl_gen = 0;

FloorCtx *find_ctx(const UhcEngine *e) {
    for (FloorCtx *c : g_fl) if (c->eng == e) return c;
    return nullptr;
}

// the hulls of a launch whose variants may be the engine's clip models, which point the tracker's envs at their run-time subjects
FloorDev with_slots(const FloorCtx *c, const UhcEngine *e) { FloorDev d = c->dev; d.slot = trackx::slot_hulls(e); return d; }

// steps 2 - 4 of floor_core.h for the warp's frame: cur / prev = the poses lanes 0 / 1 placed (prev null: no previous frame)
__device__ __forceinline__ void warp_frame(const FloorDev &d, int variant, const double *cur, const double *prev, int lane, double *out) {
    const double *v = variant < d.nshape ? d.vert + (size_t)variant * d.nvert * 3 : d.slot + (size_t)(variant - d.nshape) * d.nvert * 3;
    const floorm::Hull h{v, d.vbody, d.nvert};
    floorm::Part p;
    floorm::lane_part(h, cur, prev, lane, &p);
    for (int off = floorm::LANES / 2; off > 0; off >>= 1) {
        floorm::Part o;
        o.min_z = __shfl_xor_sync(FULL, p.min_z, off); o.below = __shfl_xor_sync(FULL, p.below, off); o.skate = __shfl_xor_sync(FULL, p.skate, off);
        o.n_below = __shfl_xor_sync(FULL, p.n_below, off); o.n_skate = __shfl_xor_sync(FULL, p.n_skate, off);
        floorm::part_merge(&p, o);
    }
    if (lane == 0) floorm::finish(p, out);
}

template <class Real>
__global__ void __launch_bounds__(32 * WARPS) k_floor_qpos(motion::MotionModel m, FloorDev d, const Real *__restrict__ qpos, long n, long pitch,
                                                           const int *__restrict__ variant, const int *__restrict__ first, bool chain,
                                                           double *__restrict__ out) {
    __shared__ double s_pose[WARPS][2][floorm::POSE_ROW];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long i = (long)blockIdx.x * WARPS + w;
    if (i >= n) return;
    const int v = variant ? variant[i] : 0;
    const bool has_prev = chain && i > 0 && !(first && first[i]);   // chain false: unrelated rows, none has a previous frame
    if (lane == 0 || (lane == 1 && has_prev)) {
        const Real *src = qpos + (size_t)(i - lane) * pitch;
        double q[motion::MQ];
        for (int k = 0; k < motion::MQ; k++) q[k] = (double)src[k];
        floorm::place(m, q, m.body + (size_t)v * motion::MB * motion::BODY6, s_pose[w][lane]);
    }
    __syncwarp();
    warp_frame(d, v, s_pose[w][0], has_prev ? s_pose[w][1] : nullptr, lane, out + (size_t)i * floorm::NCOL);
}

// frames [clip_adr[c0], clip_adr[c1]) of the dataset, nf of them; rows = the raw rows of those clips only (as k_motion_frames)
__global__ void __launch_bounds__(32 * WARPS) k_floor_motion(motion::MotionModel m, FloorDev d, int kind, int pose_dim, const double *__restrict__ rows,
                                                             const int *__restrict__ clip_adr, const int *__restrict__ fk_model, int c0, int c1, int nf,
                                                             double *__restrict__ out, double *__restrict__ feet) {
    __shared__ double s_pose[WARPS][2][floorm::POSE_ROW];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * WARPS + w;
    if (i >= nf) return;
    const int f0 = clip_adr[c0], f = f0 + i;
    int lo = c0, hi = c1 - 1;          // clip of frame f: the last clip starting at or before it
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (clip_adr[mid] <= f) lo = mid; else hi = mid - 1; }
    const int v = fk_model ? fk_model[lo] : 0, t = f - clip_adr[lo];
    const int row_w = kind == motion::KIND_QPOS ? motion::MQ : pose_dim + 3;
    const bool has_prev = t > 0;
    if (lane == 0 || (lane == 1 && has_prev)) {
        const double *body = m.body + (size_t)v * motion::MB * motion::BODY6;
        double q[motion::MQ];
        motion::m_load_qpos(m, kind, pose_dim, rows + (size_t)(i - lane) * row_w, body, q);
        floorm::place(m, q, body, s_pose[w][lane]);
        if (lane == 0 && feet)
            for (int k = 0; k < floorm::NFEET; k++) feet[(size_t)f * floorm::NFEET + k] = s_pose[w][0][render::POSE * floorm::foot_body(k) + 11];
    }
    __syncwarp();
    warp_frame(d, v, s_pose[w][0], has_prev ? s_pose[w][1] : nullptr, lane, out + (size_t)f * floorm::NCOL);
}

template <class Real>
__global__ void __launch_bounds__(32 * WARPS) k_eval_floor(motion::MotionModel m, FloorDev d, const Real *__restrict__ state, const int *__restrict__ istate,
                                                           const int *__restrict__ clip_model, const UhcEvalClip *__restrict__ clips, int *__restrict__ done,
                                                           double *__restrict__ prev, int n, int window, int slot, double *__restrict__ win_floor) {
    __shared__ double s_pose[WARPS][2][floorm::POSE_ROW];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * WARPS + w;
    if (i >= n || slot >= window) return;
    const int frames = clips[i].frames;
    if (frames <= done[i]) return;
    const int v = clip_model ? clip_model[istate[(size_t)i * SI_SIZE + SI_CLIP]] : 0;
    const bool has_prev = frames > 1;
    const Real *st = state + (size_t)i * ST_SIZE + ST_Q;
    double *pq = prev + (size_t)i * motion::MQ;
    if (lane == 0 || (lane == 1 && has_prev)) {
        double q[motion::MQ];
        for (int k = 0; k < motion::MQ; k++) q[k] = lane == 0 ? (double)st[k] : pq[k];
        floorm::place(m, q, m.body + (size_t)v * motion::MB * motion::BODY6, s_pose[w][lane]);
    }
    __syncwarp();                      // every lane has read done[i] and lane 1 prev[i]
    warp_frame(d, v, s_pose[w][0], has_prev ? s_pose[w][1] : nullptr, lane, win_floor + ((size_t)i * window + slot) * floorm::NCOL);
    for (int k = lane; k < motion::MQ; k += floorm::LANES) pq[k] = (double)st[k];
    if (lane == 0) done[i] = frames;
}

// pinned / device staging of uhc_motion_floor: two buffers, so the host fills one chunk while the device copies and reduces the other
struct Staging {
    double *h[2] = {nullptr, nullptr}, *d[2] = {nullptr, nullptr}; int *d_fk = nullptr, *d_adr = nullptr;
    cudaEvent_t ev[2] = {};            // per buffer: its kernel has ended
    ~Staging() {
        for (int s = 0; s < 2; s++) {
            if (h[s]) cudaFreeHost(h[s]);
            if (d[s]) cudaFree(d[s]);
            if (ev[s]) cudaEventDestroy(ev[s]);
        }
        if (d_fk) cudaFree(d_fk);
        if (d_adr) cudaFree(d_adr);
    }
};

}  // namespace

namespace uhc {
namespace floorm {

unsigned long long floor_gen(const UhcEngine *e) { const FloorCtx *c = find_ctx(e); return c ? c->gen : 0; }

cudaError_t launch_eval_floor(UhcEngine *e, int precision, const void *state, const int *istate, const int *clip_model, const UhcEvalClip *clips,
                              int *done, double *prev, int n, int window, int slot, double *win_floor, cudaStream_t st) {
    const FloorCtx *c = find_ctx(e);
    const motion::MotionModel &m = trackx::motion_model(e);
    const unsigned blocks = (unsigned)((n + WARPS - 1) / WARPS);
    if (precision == 32)
        k_eval_floor<float><<<blocks, 32 * WARPS, 0, st>>>(m, with_slots(c, e), (const float *)state, istate, clip_model, clips, done, prev, n, window, slot, win_floor);
    else
        k_eval_floor<double><<<blocks, 32 * WARPS, 0, st>>>(m, with_slots(c, e), (const double *)state, istate, clip_model, clips, done, prev, n, window, slot, win_floor);
    return cudaGetLastError();
}

}  // namespace floorm
}  // namespace uhc

extern "C" {

const char *uhc_floor_last_error(void) { return uhc_last_error(); }

int uhc_floor_init(UhcEngine *e, const UhcFloorHulls *h) {
    if (!e || !h || !h->hull || !h->hull_adr || !h->hull_num) { uhc_err() = "uhc_floor_init: null argument"; return -2; }
    if (h->nshape != trackx::num_shapes(e)) { uhc_err() = "uhc_floor_init: nshape differs from the engine's shape variants"; return -2; }
    if (h->nvert < 1) { uhc_err() = "uhc_floor_init: nvert < 1"; return -2; }
    std::vector<unsigned char> vbody((size_t)h->nvert);
    int next = 0;
    for (int b = 0; b < motion::MB; b++) {
        if (h->hull_adr[b] != next || h->hull_num[b] < 1 || h->hull_num[b] > h->nvert - next) {
            uhc_err() = "uhc_floor_init: hull_adr / hull_num do not tile the vertices in body order"; return -2;
        }
        for (int k = 0; k < h->hull_num[b]; k++) vbody[(size_t)next + k] = (unsigned char)b;
        next += h->hull_num[b];
    }
    if (next != h->nvert) { uhc_err() = "uhc_floor_init: hull_adr / hull_num do not tile the vertices in body order"; return -2; }
    // built aside and registered only when complete, so a failed upload leaves the engine without hulls, not with half of them
    const size_t nv = (size_t)h->nshape * h->nvert * 3;
    double *d_vert = nullptr; unsigned char *d_vbody = nullptr;
    cudaError_t ce = cudaMalloc((void **)&d_vert, nv * sizeof(double));
    if (ce == cudaSuccess) ce = cudaMalloc((void **)&d_vbody, vbody.size());
    if (ce == cudaSuccess) ce = cudaMemcpy(d_vert, h->hull, nv * sizeof(double), cudaMemcpyHostToDevice);
    if (ce == cudaSuccess) ce = cudaMemcpy(d_vbody, vbody.data(), vbody.size(), cudaMemcpyHostToDevice);
    if (ce != cudaSuccess) {
        cudaFree(d_vert); cudaFree(d_vbody);
        uhc_err() = std::string("uhc_floor_init: ") + cudaGetErrorString(ce); return -1;
    }
    uhc_floor_release(e);
    FloorCtx *c = new FloorCtx();
    c->eng = e; c->nshape = h->nshape; c->gen = ++g_fl_gen; c->d_vert = d_vert; c->d_vbody = d_vbody;
    c->dev = FloorDev{d_vert, d_vbody, h->nvert, h->nshape, nullptr};
    g_fl.push_back(c);
    return 0;
}

void uhc_floor_release(UhcEngine *e) {
    for (size_t i = 0; i < g_fl.size(); i++) if (g_fl[i]->eng == e) {
        FloorCtx *c = g_fl[i];
        if (c->d_vert) cudaFree(c->d_vert);
        if (c->d_vbody) cudaFree(c->d_vbody);
        delete c; g_fl.erase(g_fl.begin() + i); return;
    }
}

int uhc_floor_qpos(UhcEngine *e, const void *qpos_dev, int precision, long n, long qpos_pitch, const int *variant_dev_or_null,
                   const int *first_dev_or_null, double *out_dev, void *stream) {
    if (!e) { uhc_err() = "uhc_floor_qpos: null engine"; return -2; }
    if (n < 0) { uhc_err() = "uhc_floor_qpos: n < 0"; return -2; }
    if (precision != 32 && precision != 64) { uhc_err() = "uhc_floor_qpos: precision must be 32 or 64"; return -2; }
    if (qpos_pitch < 76) { uhc_err() = "uhc_floor_qpos: qpos_pitch < 76"; return -2; }
    if (n > 0 && (!qpos_dev || !out_dev)) { uhc_err() = "uhc_floor_qpos: null pointer"; return -2; }
    const FloorCtx *c = find_ctx(e);
    if (!c) { uhc_err() = "uhc_floor_qpos: no hull vertices (uhc_floor_init)"; return -2; }
    if (n == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    if (variant_dev_or_null) {
        std::vector<int> v((size_t)n);
        CK(cudaMemcpyAsync(v.data(), variant_dev_or_null, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        for (long i = 0; i < n; i++)
            if (v[(size_t)i] < 0 || v[(size_t)i] >= c->nshape) { uhc_err() = "uhc_floor_qpos: variant out of range"; return -2; }
    }
    const motion::MotionModel &m = trackx::motion_model(e);
    const unsigned blocks = (unsigned)((n + WARPS - 1) / WARPS);
    if (precision == 32)
        k_floor_qpos<float><<<blocks, 32 * WARPS, 0, st>>>(m, c->dev, (const float *)qpos_dev, n, qpos_pitch, variant_dev_or_null, first_dev_or_null, true, out_dev);
    else
        k_floor_qpos<double><<<blocks, 32 * WARPS, 0, st>>>(m, c->dev, (const double *)qpos_dev, n, qpos_pitch, variant_dev_or_null, first_dev_or_null, true, out_dev);
    CK(cudaGetLastError());
    return 0;
}

int uhc_track_floor(UhcEngine *e, const void *state_out_dev, double *out_dev, void *stream) {
    if (!e || !state_out_dev || !out_dev) { uhc_err() = "uhc_track_floor: null argument"; return -2; }
    const FloorCtx *c = find_ctx(e);
    if (!c) { uhc_err() = "uhc_track_floor: no hull vertices (uhc_floor_init)"; return -2; }
    evalx::EngineRefs R; evalx::engine_refs(e, &R);
    if (!trackx::tracking(e) || R.num_clips != R.E) { uhc_err() = "uhc_track_floor: not tracking (uhc_track_begin), or the tracker's table was replaced"; return -2; }
    const motion::MotionModel &m = trackx::motion_model(e);
    const unsigned blocks = (unsigned)((R.E + WARPS - 1) / WARPS);
    cudaStream_t st = (cudaStream_t)stream;
    if (R.precision == 32)
        k_floor_qpos<float><<<blocks, 32 * WARPS, 0, st>>>(m, with_slots(c, e), (const float *)state_out_dev, R.E, UHC_TRACK_OUT, trackx::clip_models(e), nullptr, false, out_dev);
    else
        k_floor_qpos<double><<<blocks, 32 * WARPS, 0, st>>>(m, with_slots(c, e), (const double *)state_out_dev, R.E, UHC_TRACK_OUT, trackx::clip_models(e), nullptr, false, out_dev);
    CK(cudaGetLastError());
    return 0;
}

int uhc_motion_floor(UhcEngine *e, int nclips, const int *clip_len, int kind, int pose_dim, const double *rows_host, const int *fk_model,
                     int chunk_frames, double *out_dev, double *feet_dev_or_null) {
    if (!e || nclips <= 0 || !clip_len || !rows_host || !out_dev) { uhc_err() = "uhc_motion_floor: bad argument"; return -2; }
    if (kind != UHC_MOTION_SMPL && kind != UHC_MOTION_QPOS) { uhc_err() = "uhc_motion_floor: kind must be UHC_MOTION_SMPL or UHC_MOTION_QPOS"; return -2; }
    if (kind == UHC_MOTION_SMPL ? (pose_dim != 72 && pose_dim != 156) : pose_dim != motion::MQ) {
        uhc_err() = "uhc_motion_floor: pose_dim must be 72 or 156 (UHC_MOTION_SMPL) or 76 (UHC_MOTION_QPOS)"; return -2;
    }
    if (chunk_frames < 0) { uhc_err() = "uhc_motion_floor: chunk_frames < 0"; return -2; }
    const FloorCtx *c = find_ctx(e);
    if (!c) { uhc_err() = "uhc_motion_floor: no hull vertices (uhc_floor_init)"; return -2; }
    std::vector<int> adr((size_t)nclips + 1, 0);
    long long total = 0;
    for (int i = 0; i < nclips; i++) {
        if (clip_len[i] < 1) { uhc_err() = "uhc_motion_floor: clip shorter than 1 frame"; return -2; }
        total += clip_len[i];
        if (total > 0x7fffffffLL) { uhc_err() = "uhc_motion_floor: more than 2^31 - 1 frames"; return -2; }
        adr[(size_t)i + 1] = (int)total;
        if (fk_model && (fk_model[i] < 0 || fk_model[i] >= c->nshape)) { uhc_err() = "uhc_motion_floor: fk_model index out of range"; return -2; }
    }
    const int row_w = kind == UHC_MOTION_SMPL ? pose_dim + 3 : motion::MQ;
    const int cap = chunk_frames > 0 ? chunk_frames : 32768;
    // chunks of whole clips, each of at most `cap` frames unless a single clip is longer (uhc_load_motions' rule)
    std::vector<int> cut(1, 0); size_t rows_max = 0;
    {
        long long k = 0;
        for (int i = 0; i < nclips; i++) {
            if (k > 0 && k + clip_len[i] > cap) { cut.push_back(i); rows_max = (size_t)k > rows_max ? (size_t)k : rows_max; k = 0; }
            k += clip_len[i];
        }
        cut.push_back(nclips); rows_max = (size_t)k > rows_max ? (size_t)k : rows_max;
    }
    CK(cudaDeviceSynchronize());
    Staging st;
    const size_t stage_bytes = rows_max * row_w * sizeof(double);
    for (int s = 0; s < 2; s++) {
        CK(cudaHostAlloc((void **)&st.h[s], stage_bytes, cudaHostAllocDefault)); CK(cudaMalloc((void **)&st.d[s], stage_bytes));
        CK(cudaEventCreateWithFlags(&st.ev[s], cudaEventDisableTiming));
    }
    CK(cudaMalloc((void **)&st.d_adr, adr.size() * sizeof(int)));
    CK(cudaMemcpy(st.d_adr, adr.data(), adr.size() * sizeof(int), cudaMemcpyHostToDevice));
    if (fk_model) { CK(cudaMalloc((void **)&st.d_fk, nclips * sizeof(int))); CK(cudaMemcpy(st.d_fk, fk_model, nclips * sizeof(int), cudaMemcpyHostToDevice)); }
    const motion::MotionModel &m = trackx::motion_model(e);
    const int nchunk = (int)cut.size() - 1;
    for (int k = 0; k < nchunk; k++) {
        const int s = k & 1, c0 = cut[k], c1 = cut[k + 1];
        const int f0 = adr[c0], nf = adr[c1] - f0;
        if (k >= 2) CK(cudaEventSynchronize(st.ev[s]));   // buffer s was last used by chunk k - 2
        memcpy(st.h[s], rows_host + (size_t)f0 * row_w, (size_t)nf * row_w * sizeof(double));
        CK(cudaMemcpyAsync(st.d[s], st.h[s], (size_t)nf * row_w * sizeof(double), cudaMemcpyHostToDevice, 0));
        k_floor_motion<<<(unsigned)((nf + WARPS - 1) / WARPS), 32 * WARPS, 0, 0>>>(m, c->dev, kind, pose_dim, st.d[s], st.d_adr, st.d_fk, c0, c1, nf, out_dev,
                                                                                  feet_dev_or_null);
        CK(cudaGetLastError());
        CK(cudaEventRecord(st.ev[s], 0));
    }
    CK(cudaDeviceSynchronize());
    return 0;
}

}  // extern "C"
