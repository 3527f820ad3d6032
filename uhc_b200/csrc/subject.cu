// subject.cu -- the subject body builder behind the C ABI (include/uhc_subject.h): k_subject, one block of NT threads per subject, in fp64.
// The block evaluates the 24 maps and offsets, maps the hull vertices and the mass properties, then builds the 75 x 75 joint-space inertia at
// qpos0 in shared memory (packed lower triangle), factors it (right-looking Cholesky, one column per step) and solves for the 24 invweights.
// Each item is one call of subject_core.h, so its bits do not depend on the thread that computes it.  Compiled with -fmad=false
// (uhc_b200/build.py), as its host emulation is with -ffp-contract=off.  sm_90a.
#include <cuda_runtime.h>
#include <math.h>
#include <string>
#include <vector>
#include "../../include/uhc_subject.h"
#include "errors.h"
#include "subject_core.h"
#include "subject_glue.h"

using namespace uhc;

namespace {

constexpr int NT = 256;
constexpr int CHUNK = 4096;            // subjects per launch: bounds the device copies of the outputs

struct SubDev {
    int nvert;
    int parent[subj::NB], sub_end[subj::NB], hull_adr[subj::NB], hull_num[subj::NB];
    const double *bf0, *hull0, *armature;  // shipped body_f [24][20], hull [nvert][3], armature [75]
    const int *vbody;                      // body of every hull vertex
    const double *map[3], *off[3];         // the bases of uhc_subject.h, NULL for a gender without one
};

__global__ void __launch_bounds__(NT) k_subject(SubDev d, const double *__restrict__ betas, const int *__restrict__ gender,
                                                double *__restrict__ body_f, double *__restrict__ hull, double *__restrict__ maps,
                                                int *__restrict__ bad) {
    using namespace subj;
    __shared__ double s_beta[NBETA];
    __shared__ double s_map[NB][MAPW];
    __shared__ double s_bf[NB][BODYF];
    __shared__ double s_L[NTRI];
    __shared__ double s_part[NB * 3];
    __shared__ Rest R;
    __shared__ int s_bad;
    const int row = blockIdx.x, tid = threadIdx.x, g = gender[row];
    if (tid < NBETA) s_beta[tid] = betas[(size_t)row * NBETA + tid];
    if (tid == 0) s_bad = 0;
    __syncthreads();
    if (tid < NB) {
        const int b = tid;
        eval_map(d.map[g] + (size_t)b * NTERM * MAPW, s_beta, s_map[b]);
        if (!(det3(s_map[b]) > 0.0)) atomicMax(&s_bad, b + 1);
        const double *bf = d.bf0 + b * BODYF;
        eval_offset(d.off[g] + (size_t)b * NTERM * 3, s_beta, bf, s_bf[b]);
        mass_props(s_map[b], bf, s_bf[b]);
        s_bf[b][18] = bf[18]; s_bf[b][19] = bf[19];
        for (int k = 0; k < MAPW; k++) if (maps) maps[((size_t)row * NB + b) * MAPW + k] = s_map[b][k];
    }
    __syncthreads();
    double *hv = hull + (size_t)row * d.nvert * 3;
    for (int v = tid; v < d.nvert; v += NT) apply(s_map[d.vbody[v]], d.hull0 + (size_t)v * 3, hv + (size_t)v * 3);
    if (tid == 0) {
        for (int b = 0; b < NB; b++) {
            for (int c = 0; c < 3; c++) {
                R.gpos[b][c] = b == 0 ? s_bf[0][c] : R.gpos[d.parent[b]][c] + s_bf[b][c];
                R.xipos[b][c] = R.gpos[b][c] + s_bf[b][3 + c];
            }
            R.mass[b] = s_bf[b][6];
            for (int k = 0; k < 6; k++) R.inertia[b][k] = s_bf[b][7 + k];
            R.parent[b] = d.parent[b];
            R.sub_end[b] = d.sub_end[b];
        }
    }
    __syncthreads();                   // R and the mapped hull are complete
    for (int e = tid; e < NTRI; e += NT) {
        int i = (int)((sqrt(8.0 * e + 1.0) - 1.0) * 0.5);
        while (tri(i + 1, 0) <= e) i++;
        while (tri(i, 0) > e) i--;
        s_L[e] = m_entry(R, d.armature, i, e - tri(i, 0));
    }
    __syncthreads();
    for (int k = 0; k < NV; k++) {
        if (tid == 0) chol_pivot(s_L, k);
        __syncthreads();
        for (int i = k + 1 + tid; i < NV; i += NT) chol_col(s_L, k, i);
        __syncthreads();
        const int m = NV - k - 1, cnt = m * (m + 1) / 2;       // entries (i, j), k < j <= i, as a packed triangle of side m
        for (int e = tid; e < cnt; e += NT) {
            int i = (int)((sqrt(8.0 * e + 1.0) - 1.0) * 0.5);
            while (tri(i + 1, 0) <= e) i++;
            while (tri(i, 0) > e) i--;
            chol_update(s_L, k, k + 1 + i, k + 1 + e - tri(i, 0));
        }
        __syncthreads();
    }
    if (tid < NB * 3) {
        double y[NV];
        s_part[tid] = invw_part(R, s_L, tid / 3, tid % 3, y);
    }
    __syncthreads();
    if (tid < NB) s_bf[tid][13] = (s_part[3 * tid] + s_part[3 * tid + 1] + s_part[3 * tid + 2]) / 3.0;
    __syncthreads();
    for (int e = tid; e < NB * BODYF; e += NT) {
        const int b = e / BODYF, c = e - b * BODYF;
        if (c < 14 || c > 17) body_f[(size_t)row * NB * BODYF + e] = s_bf[b][c];
    }
    if (tid < NB) {
        const int b = tid;
        double sp[4] = {0.0, 0.0, 0.0, 0.0};
        if (d.hull_num[b] > 0) sphere(hv + (size_t)d.hull_adr[b] * 3, d.hull_num[b], sp);
        for (int c = 0; c < 4; c++) body_f[((size_t)row * NB + b) * BODYF + 14 + c] = sp[c];
    }
    if (tid == 0) bad[row] = s_bad;
}

// device buffers freed on every return path
struct Bufs {
    std::vector<void *> p;
    ~Bufs() { for (void *x : p) cudaFree(x); }
    template <class T> cudaError_t alloc(T **d, size_t n) {
        void *x = nullptr;
        const cudaError_t ce = cudaMalloc(&x, n * sizeof(T) + 8);
        if (ce == cudaSuccess) p.push_back(x);
        *d = (T *)x;
        return ce;
    }
    template <class T> cudaError_t up(T **d, const T *src, size_t n) {
        cudaError_t ce = alloc(d, n);
        if (ce == cudaSuccess) ce = cudaMemcpy(*d, src, n * sizeof(T), cudaMemcpyHostToDevice);
        return ce;
    }
};

struct DeviceScope {                   // the caller's current device is restored on return
    int prev = -1;
    ~DeviceScope() { if (prev >= 0) cudaSetDevice(prev); }
};

// the builder's inputs on the current device: variant 0 of base and every gender's basis.  -2 when the hull does not tile into bodies
int prepare(const UhcModelHost *base, const UhcSubjectBasis *basis, const char *who, SubDev *d, Bufs &B) {
    using namespace subj;
    const int V = base->nvert;
    std::vector<int> vbody((size_t)V, -1);
    for (int b = 0; b < NB; b++)
        for (int k = 0; k < base->hull_num[b]; k++) {
            const long v = (long)base->hull_adr[b] + k;
            if (v < 0 || v >= V) { uhc_err() = std::string(who) + ": hull_adr / hull_num outside the hull"; return -2; }
            vbody[(size_t)v] = b;
        }
    for (int v = 0; v < V; v++)
        if (vbody[(size_t)v] < 0) { uhc_err() = std::string(who) + ": a hull vertex belongs to no body"; return -2; }
    std::vector<double> arm(NV);
    for (int i = 0; i < NV; i++) arm[(size_t)i] = base->dof_f[4 * i];
    *d = SubDev{};
    d->nvert = V;
    for (int b = 0; b < NB; b++) {
        d->parent[b] = base->parent[b]; d->sub_end[b] = base->body_sub_end[b]; d->hull_adr[b] = base->hull_adr[b]; d->hull_num[b] = base->hull_num[b];
    }
    double *bf0, *hull0, *armd; int *vb;
    CK(B.up(&bf0, base->body_f, (size_t)NB * BODYF));
    CK(B.up(&hull0, base->hull, (size_t)V * 3));
    CK(B.up(&armd, arm.data(), arm.size()));
    CK(B.up(&vb, vbody.data(), vbody.size()));
    d->bf0 = bf0; d->hull0 = hull0; d->armature = armd; d->vbody = vb;
    for (int g = 0; g < 3; g++) {
        d->map[g] = d->off[g] = nullptr;
        if (!basis->map[g]) continue;
        double *m, *o;
        CK(B.up(&m, basis->map[g], (size_t)NB * NTERM * MAPW));
        CK(B.up(&o, basis->offset[g], (size_t)NB * NTERM * 3));
        d->map[g] = m; d->off[g] = o;
    }
    return 0;
}

int run(int device, const UhcModelHost *base, const UhcSubjectBasis *basis, int n, const double *betas, const int *gender, double *body_f,
        double *hull, double *maps) {
    using namespace subj;
    const int V = base->nvert;
    DeviceScope scope;
    CK(cudaGetDevice(&scope.prev));
    CK(cudaSetDevice(device));
    Bufs B;
    SubDev d;
    if (const int rc = prepare(base, basis, "uhc_subject_bodies", &d, B)) return rc;
    const int cap = n < CHUNK ? n : CHUNK;
    double *be, *bfo, *hu, *mp = nullptr; int *ge, *bad;
    CK(B.alloc(&be, (size_t)cap * NBETA));
    CK(B.alloc(&ge, (size_t)cap));
    CK(B.alloc(&bfo, (size_t)cap * NB * BODYF));
    CK(B.alloc(&hu, (size_t)cap * V * 3));
    CK(B.alloc(&bad, (size_t)cap));
    if (maps) CK(B.alloc(&mp, (size_t)cap * NB * MAPW));
    std::vector<int> hbad((size_t)n);
    std::vector<double> bf_all((size_t)n * NB * BODYF), hull_all((size_t)n * V * 3), map_all(maps ? (size_t)n * NB * MAPW : 0);
    for (int r0 = 0; r0 < n; r0 += CHUNK) {
        const int m = n - r0 < CHUNK ? n - r0 : CHUNK;
        CK(cudaMemcpy(be, betas + (size_t)r0 * NBETA, (size_t)m * NBETA * sizeof(double), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(ge, gender + r0, (size_t)m * sizeof(int), cudaMemcpyHostToDevice));
        k_subject<<<(unsigned)m, NT>>>(d, be, ge, bfo, hu, mp, bad);
        CK(cudaGetLastError());
        CK(cudaMemcpy(hbad.data() + r0, bad, (size_t)m * sizeof(int), cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(bf_all.data() + (size_t)r0 * NB * BODYF, bfo, (size_t)m * NB * BODYF * sizeof(double), cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(hull_all.data() + (size_t)r0 * V * 3, hu, (size_t)m * V * 3 * sizeof(double), cudaMemcpyDeviceToHost));
        if (maps) CK(cudaMemcpy(map_all.data() + (size_t)r0 * NB * MAPW, mp, (size_t)m * NB * MAPW * sizeof(double), cudaMemcpyDeviceToHost));
    }
    for (int r = 0; r < n; r++)
        if (hbad[(size_t)r]) {
            uhc_err() = "uhc_subject_bodies: subject " + std::to_string(r) + ": the map of body " + std::to_string(hbad[(size_t)r] - 1) +
                        " inverts it (det A <= 0)";
            return -2;
        }
    std::copy(bf_all.begin(), bf_all.end(), body_f);
    std::copy(hull_all.begin(), hull_all.end(), hull);
    if (maps) std::copy(map_all.begin(), map_all.end(), maps);
    return 0;
}

}  // namespace

extern "C" int uhc_subject_bodies(int device, const UhcModelHost *base, const UhcSubjectBasis *basis, int n, const double *betas_host,
                                  const int *gender_host, double *body_f_host, double *hull_host, double *maps_host_or_null) {
    using namespace subj;
    if (!base || !basis) { uhc_err() = "uhc_subject_bodies: null pointer"; return -2; }
    if (n < 0) { uhc_err() = "uhc_subject_bodies: n < 0"; return -2; }
    if (n == 0) return 0;
    if (!betas_host || !gender_host || !body_f_host || !hull_host || !base->body_f || !base->hull || !base->dof_f || !base->hull_adr ||
        !base->hull_num || !base->parent || !base->body_sub_end || base->nvert < 1) {
        uhc_err() = "uhc_subject_bodies: null pointer"; return -2;
    }
    for (int g = 0; g < 3; g++)
        if (!basis->map[g] != !basis->offset[g]) { uhc_err() = "uhc_subject_bodies: gender " + std::to_string(g) + " has one of its two bases"; return -2; }
    for (int r = 0; r < n; r++) {
        const int g = gender_host[r];
        if (g < 0 || g > 2) { uhc_err() = "uhc_subject_bodies: subject " + std::to_string(r) + ": gender code outside 0 .. 2"; return -2; }
        if (!basis->map[g]) { uhc_err() = "uhc_subject_bodies: subject " + std::to_string(r) + ": gender " + std::to_string(g) + " has no model"; return -2; }
        for (int l = 0; l < NBETA; l++)
            if (!isfinite(betas_host[(size_t)r * NBETA + l])) { uhc_err() = "uhc_subject_bodies: subject " + std::to_string(r) + ": non-finite beta"; return -2; }
    }
    return run(device, base, basis, n, betas_host, gender_host, body_f_host, hull_host, maps_host_or_null);
}

// ---- the builder of the tracker's run-time subjects (subject_glue.h): k_subject over rows already on the device
struct uhc::subjx::Builder {
    SubDev d;
    Bufs B;
};

int uhc::subjx::builder_create(const UhcModelHost *base, const UhcSubjectBasis *basis, const char *who, Builder **out) {
    if (!base || !basis || !base->body_f || !base->hull || !base->dof_f || !base->hull_adr || !base->hull_num || !base->parent ||
        !base->body_sub_end || base->nvert < 1) {
        uhc_err() = std::string(who) + ": null pointer"; return -2;
    }
    for (int g = 0; g < 3; g++)
        if (!basis->map[g] != !basis->offset[g]) { uhc_err() = std::string(who) + ": gender " + std::to_string(g) + " has one of its two bases"; return -2; }
    if (!basis->map[0] && !basis->map[1] && !basis->map[2]) { uhc_err() = std::string(who) + ": the basis has no gender"; return -2; }
    Builder *b = new Builder();
    if (const int rc = prepare(base, basis, who, &b->d, b->B)) { delete b; return rc; }
    *out = b;
    return 0;
}

void uhc::subjx::builder_free(Builder *b) { delete b; }
bool uhc::subjx::has_gender(const Builder *b, int g) { return g >= 0 && g < 3 && b->d.map[g] != nullptr; }
int uhc::subjx::nvert(const Builder *b) { return b->d.nvert; }

cudaError_t uhc::subjx::launch(const Builder *b, int n, const double *betas, const int *gender, double *body_f, double *hull, int *bad, cudaStream_t st) {
    k_subject<<<(unsigned)n, NT, 0, st>>>(b->d, betas, gender, body_f, hull, nullptr, bad);
    return cudaGetLastError();
}
