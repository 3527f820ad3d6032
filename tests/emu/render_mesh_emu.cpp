// render_mesh_emu.cpp -- TEST INFRASTRUCTURE: compiles the mesh renderer's refit and pixel path (uhc_b200/csrc/render_mesh_core.h) as host
// code (-DUHC_EMU, -ffp-contract=off) so the kernels' arithmetic is checked against an independent fp64 ray caster on a CPU-only box, and
// the GPU's pixels against these bit for bit.  Never loaded by the product path (uhc_b200/engine.py only loads the CUDA library).
#define UHC_EMU 1
#define UHC_RENDER_HOST 1
#include <string.h>
#include <vector>
#include "../../include/uhc_b200.h"
#include "../../include/uhc_render.h"
#include "../../uhc_b200/csrc/render_mesh_core.h"

using namespace uhc;

extern "C" {
// uhc_render_mesh_init's table checks: 0, or -2 with the reason in why
int emu_render_mesh_check(const UhcRenderMesh *m, char *why, int cap) {
    const char *w = "";
    const int rc = render::mesh_tables_check(*m, &w);
    strncpy(why, w, (size_t)cap - 1);
    why[cap - 1] = 0;
    return rc;
}

// uhc_render_mesh on the host: verts / ghost [n][nvert][3], root [n][3] (or NULL), the topology m; boxes_out (or NULL) = [n][48 + 2 nleaf][6],
// the refitted boxes in the device's scratch layout (the ghost half left untouched without a ghost)
void emu_render_mesh(const UhcRenderCamera *cam, int W, int H, long n, const float *verts, const float *ghost, const float *root,
                     const UhcRenderMesh *m, unsigned char *rgb, float *depth, unsigned char *label, float *boxes_out) {
    const int nh = ghost ? 2 : 1, SL = 2 * render::NB, nleaf = m->nleaf;
    const size_t fbox = (size_t)(SL + 2 * nleaf) * 6;
    render::Cam c;
    render::camera_setup(*cam, W, H, nh, &c);
    std::vector<float> box(fbox);
    for (long f = 0; f < n; f++) {
        for (int h = 0; h < nh; h++) {
            const float *v = (h ? ghost : verts) + (size_t)f * m->nvert * 3;
            float *leaf = box.data() + SL * 6 + (size_t)h * nleaf * 6;
            for (int l = 0; l < nleaf; l++) render::refit_leaf(v, m->face, m->leaf_first[l], m->leaf_first[l + 1], h, c.shift, leaf + 6 * l);
            for (int b = 0; b < render::NB; b++) render::union_boxes(leaf, m->body_leaf[b], m->body_leaf[b + 1], box.data() + 6 * (h * render::NB + b));
        }
        if (boxes_out) {
            float *o = boxes_out + (size_t)f * fbox;
            for (int k = 0; k < nh * render::NB * 6; k++) o[k] = box[k];
            for (int k = 0; k < nh * nleaf * 6; k++) o[SL * 6 + k] = box[SL * 6 + k];
        }
        render::MeshScene s;
        s.verts[0] = verts + (size_t)f * m->nvert * 3;
        s.verts[1] = ghost ? ghost + (size_t)f * m->nvert * 3 : s.verts[0];
        s.face = m->face; s.leaf_first = m->leaf_first; s.body_leaf = m->body_leaf;
        s.body_box = box.data(); s.leaf_box = box.data() + SL * 6;
        s.nleaf = nleaf; s.visible = c.visible; s.shift = c.shift;
        s.root = root ? root + 3 * (size_t)f : nullptr;
        for (int y = 0; y < H; y++)
            for (int x = 0; x < W; x++) {
                const size_t px = ((size_t)f * H + y) * W + x;
                render::shade_pixel(c, s, x, y, W, H, rgb + 3 * px, depth ? depth + px : nullptr, label ? label + px : nullptr);
            }
    }
}
}
