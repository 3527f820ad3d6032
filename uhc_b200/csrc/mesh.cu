// mesh.cu -- SMPL linear blend skinning behind the C ABI (include/uhc_mesh.h):
//   k_shape_joints  per shape row and joint: J = J_regressor . (v_template + shapedirs . beta), fp64, a fixed tree over the vertices
//   k_shape_verts   per shape row and vertex: v_shaped, fp64 rounded once to fp32
//   k_rows          per row: mesh_core.h row_chain (fp64) -> the pose feature and A_k in fp32 scratch, the posed joints
//   k_mesh<FLOOR>   a tile of TS consecutive rows x NT vertices: the 207-term pose blend (posedirs read once per tile and used for every row
//                   of it), the skinning sum over the vertex's non-zero weights, + trans in fp64.  FLOOR = false writes the vertices; FLOOR =
//                   true reduces them against the floor (floor_core.h's columns) and writes nothing else: its slot 0 is the predecessor of
//                   the tile's first row, recomputed, so every row's previous vertices are at hand.
// Every fp32 operation of the vertex path is an explicit _rn intrinsic, so a row's vertices are the same bits in either kernel and in every
// slot of a tile.  Compiled with -fmad=false (uhc_b200/build.py), which leaves the intrinsics as written.  sm_90a.
#include <cuda_runtime.h>
#include <math.h>
#include <string>
#include <vector>
#include "../../include/uhc_floor.h"
#include "../../include/uhc_mesh.h"
#include "engine_slots.h"
#include "errors.h"
#include "floor_core.h"
#include "mesh_core.h"

using namespace uhc;

namespace {

constexpr int NT = 128;                // threads per block, one vertex each
constexpr int WARPS = NT / 32;
constexpr int TS = 16;                 // row slots of a tile
constexpr long CHUNK = 32768;          // rows per pass through the per-row scratch
constexpr int AJ = meshm::NJ * meshm::AROW;
constexpr unsigned FULL = 0xffffffffu;

struct MeshDev {
    int V;
    int parents[meshm::NJ];
    const double *vt, *sd, *jreg;      // [V][3], [V][3][10], [24][V]
    const float *pd;                   // [207][V][3]
    const int *w_adr, *w_j;            // the non-zero weights of vertex v: entries w_adr[v] .. w_adr[v + 1] - 1, in joint order
    const float *w_w;
};

struct MeshCtx {
    MeshDev dev{};
    void *own[7] = {};                 // the model's device arrays
    float *vs = nullptr; double *J = nullptr; int cap_nb = 0;        // shape scratch: [nb][V][3], [nb][24][3]
    float *pf = nullptr, *A = nullptr; long cap_rows = 0;             // row scratch: [rows][207], [rows][24][12]
    ~MeshCtx() {
        for (void *p : own) if (p) cudaFree(p);
        if (vs) cudaFree(vs);
        if (J) cudaFree(J);
        if (pf) cudaFree(pf);
        if (A) cudaFree(A);
    }
};
MeshCtx *find_ctx(const UhcEngine *e) { return (MeshCtx *)engine_slot(e, SLOT_MESH); }

__device__ __forceinline__ double shaped(const MeshDev &d, long v, int c, const double *beta) {
    const double *s = d.sd + ((size_t)v * 3 + c) * meshm::NBETA;
    double x = d.vt[(size_t)v * 3 + c];
    for (int l = 0; l < meshm::NBETA; l++) x = x + s[l] * beta[l];
    return x;
}

__global__ void __launch_bounds__(256) k_shape_joints(MeshDev d, const double *__restrict__ betas, double *__restrict__ J) {
    __shared__ double red[3][256];
    const int j = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const double *beta = betas + (size_t)b * meshm::NBETA;
    double s[3] = {0.0, 0.0, 0.0};
    for (long v = tid; v < d.V; v += 256) {
        const double w = d.jreg[(size_t)j * d.V + v];
        for (int c = 0; c < 3; c++) s[c] = s[c] + w * shaped(d, v, c, beta);
    }
    for (int c = 0; c < 3; c++) red[c][tid] = s[c];
    __syncthreads();
    for (int h = 128; h > 0; h >>= 1) {
        if (tid < h) for (int c = 0; c < 3; c++) red[c][tid] = red[c][tid] + red[c][tid + h];
        __syncthreads();
    }
    if (tid < 3) J[((size_t)b * meshm::NJ + j) * 3 + tid] = red[tid][0];
}

__global__ void __launch_bounds__(256) k_shape_verts(MeshDev d, const double *__restrict__ betas, int nb, float *__restrict__ vs) {
    const long i = (long)blockIdx.x * 256 + threadIdx.x;
    if (i >= (long)nb * d.V) return;
    const long b = i / d.V, v = i - b * d.V;
    for (int c = 0; c < 3; c++) vs[(size_t)i * 3 + c] = (float)shaped(d, v, c, betas + (size_t)b * meshm::NBETA);
}

// scratch slot s holds row r_lo + s (r_lo = the chunk's first row - 1, so a floor tile finds its first row's predecessor); joints are written
// for rows >= r_out only
__global__ void __launch_bounds__(128) k_rows(MeshDev d, const double *__restrict__ pose, const double *__restrict__ trans,
                                              const int *__restrict__ beta_idx, const double *__restrict__ J, long r_lo, long m, long r_out,
                                              float *__restrict__ pf, float *__restrict__ A, double *__restrict__ joints) {
    const long s = (long)blockIdx.x * 128 + threadIdx.x;
    const long row = r_lo + s;
    if (s >= m || row < 0) return;
    const int b = beta_idx ? beta_idx[row] : 0;
    meshm::row_chain(d.parents, pose + (size_t)row * 72, J + (size_t)b * meshm::NJ * 3, trans + (size_t)row * 3, pf + (size_t)s * meshm::NPF,
                     A + (size_t)s * AJ, joints && row >= r_out ? joints + (size_t)row * meshm::NJ * 3 : nullptr);
}

// rows c0 .. c1 - 1 of this chunk; scratch slot of a row = row - (c0 - 1).  FLOOR: tiles of TS - 1 rows, slot 0 = the first row's predecessor.
template <bool FLOOR>
__global__ void __launch_bounds__(NT) k_mesh(MeshDev d, const float *__restrict__ vs, const float *__restrict__ pf, const float *__restrict__ A,
                                             const double *__restrict__ trans, const int *__restrict__ beta_idx, const int *__restrict__ first,
                                             long c0, long c1, float *__restrict__ verts, double *__restrict__ out) {
    __shared__ __align__(16) float s_pf[meshm::NPF][TS];
    __shared__ float s_A[TS][AJ];
    __shared__ double s_tr[TS][3];
    __shared__ int s_b[TS], s_prev[TS];
    __shared__ floorm::Part s_acc[WARPS][TS];
    constexpr int F = FLOOR ? 1 : 0;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const long r0 = c0 + (long)blockIdx.x * (TS - F) - F;    // row of slot 0
    const long r_lo = c0 - 1;
    auto live = [&](long row) { return row >= 0 && row >= r_lo && row < c1; };
    for (int i = tid; i < meshm::NPF * TS; i += NT) {
        const int s = i % TS, j = i / TS;
        const long row = r0 + s;
        s_pf[j][s] = live(row) ? pf[(size_t)(row - r_lo) * meshm::NPF + j] : 0.0f;
    }
    for (int i = tid; i < TS * AJ; i += NT) {
        const int s = i / AJ, k = i - s * AJ;
        const long row = r0 + s;
        s_A[s][k] = live(row) ? A[(size_t)(row - r_lo) * AJ + k] : 0.0f;
    }
    if (tid < TS) {
        const long row = r0 + tid;
        const bool ok = live(row);
        s_b[tid] = ok ? (beta_idx ? beta_idx[row] : 0) : -1;
        for (int c = 0; c < 3; c++) s_tr[tid][c] = ok ? trans[(size_t)row * 3 + c] : 0.0;
        s_prev[tid] = ok && row > 0 && !(first && first[row]);
    }
    if (FLOOR)
        for (int i = tid; i < WARPS * TS; i += NT) {
            floorm::Part &p = s_acc[i / TS][i % TS];
            p.min_z = floorm::HUGE_Z; p.below = 0.0; p.skate = 0.0; p.n_below = 0; p.n_skate = 0;
        }
    __syncthreads();
    const long V = d.V;
    for (long vb = (long)blockIdx.y * NT; vb < V; vb += (long)gridDim.y * NT) {
        const long v = vb + tid;
        const bool ok = v < V;
        float acc[TS][3];
#pragma unroll
        for (int s = 0; s < TS; s++) acc[s][0] = acc[s][1] = acc[s][2] = 0.0f;
        if (ok) {
            const float *p = d.pd + (size_t)v * 3;
            const size_t step = (size_t)V * 3;
#pragma unroll 3
            for (int j = 0; j < meshm::NPF; j++) {
                const float p0 = __ldg(p), p1 = __ldg(p + 1), p2 = __ldg(p + 2);
                p += step;
                const float4 *f = reinterpret_cast<const float4 *>(s_pf[j]);
#pragma unroll
                for (int q = 0; q < TS / 4; q++) {
                    const float4 x = f[q];
                    const float xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
                    for (int u = 0; u < 4; u++) {
                        acc[4 * q + u][0] = __fmaf_rn(xs[u], p0, acc[4 * q + u][0]);
                        acc[4 * q + u][1] = __fmaf_rn(xs[u], p1, acc[4 * q + u][1]);
                        acc[4 * q + u][2] = __fmaf_rn(xs[u], p2, acc[4 * q + u][2]);
                    }
                }
            }
        }
        const int e0 = ok ? d.w_adr[v] : 0, e1 = ok ? d.w_adr[v + 1] : 0;
#pragma unroll
        for (int s = 0; s < TS; s++) {
            const int b = s_b[s];
            if (!ok || b < 0) continue;
            const float *sv = vs + ((size_t)b * V + v) * 3;
            const float x = __fadd_rn(acc[s][0], sv[0]), y = __fadd_rn(acc[s][1], sv[1]), z = __fadd_rn(acc[s][2], sv[2]);
            float T[meshm::AROW];
#pragma unroll
            for (int i = 0; i < meshm::AROW; i++) T[i] = 0.0f;
            for (int e = e0; e < e1; e++) {
                const float wt = d.w_w[e];
                const float *a = s_A[s] + meshm::AROW * d.w_j[e];
#pragma unroll
                for (int i = 0; i < meshm::AROW; i++) T[i] = __fmaf_rn(wt, a[i], T[i]);
            }
#pragma unroll
            for (int c = 0; c < 3; c++) {
                const float r = __fmaf_rn(T[4 * c], x, __fmaf_rn(T[4 * c + 1], y, __fmaf_rn(T[4 * c + 2], z, T[4 * c + 3])));
                acc[s][c] = __double2float_rn(__dadd_rn((double)r, s_tr[s][c]));
            }
        }
        if (!FLOOR) {
#pragma unroll
            for (int s = 0; s < TS; s++)
                if (ok && s_b[s] >= 0)
                    for (int c = 0; c < 3; c++) verts[((size_t)(r0 + s) * V + v) * 3 + c] = acc[s][c];
        } else {
#pragma unroll
            for (int s = 1; s < TS; s++) {
                floorm::Part p; p.min_z = floorm::HUGE_Z; p.below = 0.0; p.skate = 0.0; p.n_below = 0; p.n_skate = 0;
                if (ok && s_b[s] >= 0) {
                    const double z = (double)acc[s][2];
                    p.min_z = z;
                    if (z < 0.0) { p.below = z; p.n_below = 1; }
                    if (s_prev[s] && z <= 0.0 && (double)acc[s - 1][2] <= 0.0) {
                        const double dx = (double)acc[s][0] - (double)acc[s - 1][0], dy = (double)acc[s][1] - (double)acc[s - 1][1];
                        p.skate = sqrt(dx * dx + dy * dy); p.n_skate = 1;
                    }
                }
                for (int off = 16; off > 0; off >>= 1) {
                    floorm::Part o;
                    o.min_z = __shfl_xor_sync(FULL, p.min_z, off); o.below = __shfl_xor_sync(FULL, p.below, off); o.skate = __shfl_xor_sync(FULL, p.skate, off);
                    o.n_below = __shfl_xor_sync(FULL, p.n_below, off); o.n_skate = __shfl_xor_sync(FULL, p.n_skate, off);
                    floorm::part_merge(&p, o);
                }
                if (lane == 0) floorm::part_merge(&s_acc[w][s], p);
            }
        }
    }
    if (FLOOR) {
        __syncthreads();
        if (tid >= 1 && tid < TS && s_b[tid] >= 0) {
            floorm::Part p = s_acc[0][tid];
            for (int k = 1; k < WARPS; k++) floorm::part_merge(&p, s_acc[k][tid]);
            floorm::finish(p, out + (size_t)(r0 + tid) * floorm::NCOL);
        }
    }
}

template <class T> cudaError_t dev_copy(T **dst, const T *src, size_t n) {
    cudaError_t ce = cudaMalloc((void **)dst, n * sizeof(T) + 4);
    if (ce == cudaSuccess) ce = cudaMemcpy(*dst, src, n * sizeof(T), cudaMemcpyHostToDevice);
    return ce;
}

// the checks and set-up both entry points share: argument checks (-2), the scratch, the shape pass
int prepare(UhcEngine *e, long n, const double *pose, const double *trans, int nb, const double *betas, const int *beta_idx, cudaStream_t st,
            const char *who, MeshCtx **out) {
    if (!e) { uhc_err() = std::string(who) + ": null engine"; return -2; }
    if (n < 0) { uhc_err() = std::string(who) + ": n < 0"; return -2; }
    if (nb < 1) { uhc_err() = std::string(who) + ": nbetas < 1"; return -2; }
    if (n > 0 && (!pose || !trans || !betas)) { uhc_err() = std::string(who) + ": null pointer"; return -2; }
    MeshCtx *c = find_ctx(e);
    if (!c) { uhc_err() = std::string(who) + ": no SMPL model (uhc_mesh_init)"; return -2; }
    *out = c;
    if (n == 0) return 0;
    if (beta_idx) {
        std::vector<int> b((size_t)n);
        CK(cudaMemcpyAsync(b.data(), beta_idx, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        for (long i = 0; i < n; i++)
            if (b[(size_t)i] < 0 || b[(size_t)i] >= nb) { uhc_err() = std::string(who) + ": beta_idx out of range"; return -2; }
    }
    const size_t V = (size_t)c->dev.V;
    if (c->cap_nb < nb) {
        CK(cudaStreamSynchronize(st));
        if (c->vs) cudaFree(c->vs);
        if (c->J) cudaFree(c->J);
        c->vs = nullptr; c->J = nullptr; c->cap_nb = 0;
        CK(cudaMalloc((void **)&c->vs, (size_t)nb * V * 3 * sizeof(float)));
        CK(cudaMalloc((void **)&c->J, (size_t)nb * meshm::NJ * 3 * sizeof(double)));
        c->cap_nb = nb;
    }
    const long rows = (n < CHUNK ? n : CHUNK) + 1;
    if (c->cap_rows < rows) {
        CK(cudaStreamSynchronize(st));
        if (c->pf) cudaFree(c->pf);
        if (c->A) cudaFree(c->A);
        c->pf = nullptr; c->A = nullptr; c->cap_rows = 0;
        CK(cudaMalloc((void **)&c->pf, (size_t)rows * meshm::NPF * sizeof(float)));
        CK(cudaMalloc((void **)&c->A, (size_t)rows * AJ * sizeof(float)));
        c->cap_rows = rows;
    }
    k_shape_joints<<<dim3(meshm::NJ, (unsigned)nb), 256, 0, st>>>(c->dev, betas, c->J);
    CK(cudaGetLastError());
    k_shape_verts<<<(unsigned)(((size_t)nb * V + 255) / 256), 256, 0, st>>>(c->dev, betas, nb, c->vs);
    CK(cudaGetLastError());
    return 0;
}

}  // namespace

extern "C" {

const char *uhc_mesh_last_error(void) { return uhc_last_error(); }

int uhc_mesh_init(UhcEngine *e, const UhcSmplModel *m) {
    if (!e || !m || !m->v_template || !m->shapedirs || !m->posedirs || !m->J_regressor || !m->weights || !m->parents) {
        uhc_err() = "uhc_mesh_init: null argument"; return -2;
    }
    if (m->nvert < 1) { uhc_err() = "uhc_mesh_init: nvert < 1"; return -2; }
    if (m->parents[0] != -1) { uhc_err() = "uhc_mesh_init: parents[0] must be -1"; return -2; }
    for (int k = 1; k < meshm::NJ; k++)
        if (m->parents[k] < 0 || m->parents[k] >= k) { uhc_err() = "uhc_mesh_init: parents[k] must lie in 0 .. k - 1"; return -2; }
    const size_t V = (size_t)m->nvert;
    auto finite = [](const double *x, size_t k) { for (size_t i = 0; i < k; i++) if (!isfinite(x[i])) return false; return true; };
    if (!finite(m->v_template, V * 3) || !finite(m->shapedirs, V * 3 * meshm::NBETA) || !finite(m->posedirs, V * 3 * meshm::NPF) ||
        !finite(m->J_regressor, V * meshm::NJ) || !finite(m->weights, V * meshm::NJ)) {
        uhc_err() = "uhc_mesh_init: non-finite value"; return -2;
    }
    std::vector<float> pd((size_t)meshm::NPF * V * 3);
    for (size_t v = 0; v < V; v++)
        for (int c = 0; c < 3; c++)
            for (int j = 0; j < meshm::NPF; j++) pd[((size_t)j * V + v) * 3 + c] = (float)m->posedirs[(v * 3 + c) * meshm::NPF + j];
    std::vector<int> adr(V + 1, 0), wj; std::vector<float> ww;
    for (size_t v = 0; v < V; v++) {
        for (int k = 0; k < meshm::NJ; k++)
            if (m->weights[v * meshm::NJ + k] != 0.0) { wj.push_back(k); ww.push_back((float)m->weights[v * meshm::NJ + k]); }
        adr[v + 1] = (int)wj.size();
    }
    // built aside and registered only when complete, so a failed upload leaves the previous model in place
    MeshCtx *c = new MeshCtx();
    double *vt = nullptr, *sd = nullptr, *jr = nullptr; float *pdd = nullptr, *w_w = nullptr; int *w_adr = nullptr, *w_j = nullptr;
    cudaError_t ce = dev_copy(&vt, m->v_template, V * 3);
    c->own[0] = vt;
    if (ce == cudaSuccess) { ce = dev_copy(&sd, m->shapedirs, V * 3 * meshm::NBETA); c->own[1] = sd; }
    if (ce == cudaSuccess) { ce = dev_copy(&jr, m->J_regressor, V * meshm::NJ); c->own[2] = jr; }
    if (ce == cudaSuccess) { ce = dev_copy(&pdd, pd.data(), pd.size()); c->own[3] = pdd; }
    if (ce == cudaSuccess) { ce = dev_copy(&w_adr, adr.data(), adr.size()); c->own[4] = w_adr; }
    if (ce == cudaSuccess) { ce = dev_copy(&w_j, wj.data(), wj.size()); c->own[5] = w_j; }
    if (ce == cudaSuccess) { ce = dev_copy(&w_w, ww.data(), ww.size()); c->own[6] = w_w; }
    if (ce != cudaSuccess) {
        delete c;
        uhc_err() = std::string("uhc_mesh_init: ") + cudaGetErrorString(ce); return -1;
    }
    uhc_mesh_release(e);
    c->dev.V = m->nvert;
    for (int k = 0; k < meshm::NJ; k++) c->dev.parents[k] = m->parents[k];
    c->dev.vt = vt; c->dev.sd = sd; c->dev.jreg = jr; c->dev.pd = pdd; c->dev.w_adr = w_adr; c->dev.w_j = w_j; c->dev.w_w = w_w;
    engine_slot(e, SLOT_MESH) = c;
    return 0;
}

void uhc_mesh_release(UhcEngine *e) {
    if (!e) return;
    delete find_ctx(e); engine_slot(e, SLOT_MESH) = nullptr;
}

int uhc_smpl_mesh(UhcEngine *e, long n, const double *pose_dev, const double *trans_dev, int nbetas, const double *betas_dev,
                  const int *beta_idx_dev_or_null, float *verts_dev_or_null, double *joints_dev_or_null, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    MeshCtx *c = nullptr;
    const int rc = prepare(e, n, pose_dev, trans_dev, nbetas, betas_dev, beta_idx_dev_or_null, st, "uhc_smpl_mesh", &c);
    if (rc || n == 0) return rc;
    const unsigned vblocks = (unsigned)((c->dev.V + NT - 1) / NT);
    for (long c0 = 0; c0 < n; c0 += CHUNK) {
        const long c1 = c0 + CHUNK < n ? c0 + CHUNK : n;
        k_rows<<<(unsigned)((c1 - c0 + 1 + 127) / 128), 128, 0, st>>>(c->dev, pose_dev, trans_dev, beta_idx_dev_or_null, c->J, c0 - 1, c1 - c0 + 1, c0,
                                                                      c->pf, c->A, joints_dev_or_null);
        CK(cudaGetLastError());
        if (verts_dev_or_null) {
            k_mesh<false><<<dim3((unsigned)((c1 - c0 + TS - 1) / TS), vblocks), NT, 0, st>>>(c->dev, c->vs, c->pf, c->A, trans_dev, beta_idx_dev_or_null,
                                                                                           nullptr, c0, c1, verts_dev_or_null, nullptr);
            CK(cudaGetLastError());
        }
    }
    return 0;
}

int uhc_smpl_floor(UhcEngine *e, long n, const double *pose_dev, const double *trans_dev, int nbetas, const double *betas_dev,
                   const int *beta_idx_dev_or_null, const int *first_dev_or_null, double *out_dev, void *stream) {
    if (n > 0 && !out_dev) { uhc_err() = "uhc_smpl_floor: null pointer"; return -2; }
    cudaStream_t st = (cudaStream_t)stream;
    MeshCtx *c = nullptr;
    const int rc = prepare(e, n, pose_dev, trans_dev, nbetas, betas_dev, beta_idx_dev_or_null, st, "uhc_smpl_floor", &c);
    if (rc || n == 0) return rc;
    for (long c0 = 0; c0 < n; c0 += CHUNK) {
        const long c1 = c0 + CHUNK < n ? c0 + CHUNK : n;
        k_rows<<<(unsigned)((c1 - c0 + 1 + 127) / 128), 128, 0, st>>>(c->dev, pose_dev, trans_dev, beta_idx_dev_or_null, c->J, c0 - 1, c1 - c0 + 1, c0,
                                                                      c->pf, c->A, nullptr);
        CK(cudaGetLastError());
        k_mesh<true><<<dim3((unsigned)((c1 - c0 + TS - 2) / (TS - 1)), 1), NT, 0, st>>>(c->dev, c->vs, c->pf, c->A, trans_dev, beta_idx_dev_or_null,
                                                                                        first_dev_or_null, c0, c1, nullptr, out_dev);
        CK(cudaGetLastError());
    }
    return 0;
}

}  // extern "C"
