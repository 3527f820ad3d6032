// render_emu.cpp -- TEST INFRASTRUCTURE: compiles the renderer's pose pass and pixel path (uhc_b200/csrc/render_core.h) as host code
// (-DUHC_EMU, -ffp-contract=off) so the kernels' arithmetic is checked against an independent fp64 ray caster on a CPU-only box, and the
// GPU's pixels against these bit for bit.  Never loaded by the product path (uhc_b200/engine.py only loads the CUDA library).
#define UHC_EMU 1
#define UHC_RENDER_HOST 1
#include <vector>
#include "../../include/uhc_b200.h"
#include "../../include/uhc_render.h"
#include "../../uhc_b200/csrc/render_core.h"

using namespace uhc;

extern "C" {
// n frames of one humanoid: qpos rows (pitch doubles apart) -> pose [n][24][12] fp32 and, when given, the fp64 FK wpos [n][72], wq [n][96].
// body_f = [nshape][24][20] of the shape variants, variant per frame (NULL: 0), parent / ee = the model's tables.
void emu_render_pose(long n, const double *qpos, long pitch, const double *body_f, int nshape, const int *variant, const int *parent, const int *ee,
                     float *pose, double *wpos_out, double *wq_out) {
    std::vector<double> body((size_t)nshape * motion::MB * motion::BODY6);
    motion::motion_body_table(body_f, UHC_BODYF, nshape, body.data());
    motion::MotionModel m;
    motion::motion_model_init(m, parent, ee, body.data());
    for (long i = 0; i < n; i++) {
        double wpos[3 * motion::MB], wq[4 * motion::MB];
        render::pose_fk(m, qpos + (size_t)i * pitch, body.data() + (size_t)(variant ? variant[i] : 0) * motion::MB * motion::BODY6, wpos, wq);
        render::pose_rows<float>(wpos, wq, pose + (size_t)i * render::NB * render::POSE);
        if (wpos_out) for (int k = 0; k < 3 * motion::MB; k++) wpos_out[(size_t)i * 3 * motion::MB + k] = wpos[k];
        if (wq_out) for (int k = 0; k < 4 * motion::MB; k++) wq_out[(size_t)i * 4 * motion::MB + k] = wq[k];
    }
}

// uhc_render_bodies on the host: pose [n][2][24][12], planes / spheres as uhc_render_init takes them (rounded to fp32 the same way)
void emu_render_bodies(const UhcRenderCamera *cam, int W, int H, long n, const float *pose, int humanoids, const int *variant, const double *plane,
                       int nplane, const int *adr, const int *num, const double *sphere, unsigned char *rgb, float *depth, unsigned char *label) {
    render::Cam c;
    render::camera_setup(*cam, W, H, humanoids, &c);
    std::vector<float> pl((size_t)nplane * 4), s_pose(2 * render::NB * render::POSE), s_sph(2 * render::NB * 4);
    for (long f = 0; f < n; f++) {
        const int v = variant ? variant[f] : 0;
        for (size_t k = 0; k < pl.size(); k++) pl[k] = (float)plane[(size_t)v * nplane * 4 + k];
        for (int j = 0; j < humanoids * render::NB; j++) {
            const int h = j / render::NB, b = j % render::NB;
            float cs[4];
            for (int k = 0; k < 4; k++) cs[k] = (float)sphere[((size_t)v * render::NB + b) * 4 + k];
            render::stage_body(pose + ((size_t)f * 2 + h) * render::NB * render::POSE + b * render::POSE, cs, h, c.shift,
                               s_pose.data() + j * render::POSE, s_sph.data() + 4 * j);
        }
        render::Scene s;
        s.plane = pl.data(); s.adr = adr; s.num = num; s.pose = s_pose.data(); s.sph = s_sph.data(); s.visible = c.visible;
        for (int y = 0; y < H; y++)
            for (int x = 0; x < W; x++) {
                const size_t px = ((size_t)f * H + y) * W + x;
                render::shade_pixel(c, s, x, y, W, H, rgb + 3 * px, depth ? depth + px : nullptr, label ? label + px : nullptr);
            }
    }
}
}
