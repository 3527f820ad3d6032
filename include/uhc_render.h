/* uhc_render.h -- C ABI of the offline renderer (part of libuhc_b200.so): the simulated and the reference humanoid drawn on the GPU as an exact
 * ray cast of the 24 convex body hulls the contact pass collides with, over a checkered floor; or, with uhc_render_mesh, as a ray cast of the
 * skinned SMPL mesh (include/uhc_mesh.h's vertices) under the same camera, floor, shading and outputs.
 *
 * Reference interface replaced: CopycatVisualizer (uhc/utils/copycat_visualizer.py) with render_video, which replays eval_seq's `pred` beside
 * `gt` in one MuJoCo scene and reads 1920x1080 frames back from the GL viewer.  The camera is MuJoCo's free camera as the visualizer sets it
 * (setup_viewing_angle: lookat z 1, azimuth 45, elevation -8, distance 5; update_pose's focus / hide_im / hide_expert / shift_expert).
 * Pointers suffixed _dev are CUDA device pointers.  Every call returns 0 on success, -2 on a bad argument (nothing is launched and the engine
 * stays usable), -1 on a CUDA error (uhc_last_error()).  Pixel indices are size_t: n * H * W * 3 may exceed 2^31.
 */
#ifndef UHC_RENDER_H
#define UHC_RENDER_H
#include "uhc_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

#define UHC_RENDER_POSE 12        /* floats per body of a pose table: row-major 3x3 rotation (body -> world), then the body origin */
#define UHC_RENDER_MAX_PLANES 512 /* face planes of one body hull, at most */

/* Face planes of the body hulls of every shape variant, in body frame: n . x + d <= 0 inside (scipy ConvexHull.equations, coplanar faces
 * merged).  Body b of variant s owns planes plane[s][plane_adr[b] .. plane_adr[b] + plane_num[b] - 1]; sphere[s][b] = centre (body frame)
 * and radius of a sphere that holds the hull (body_f columns 14:18).  Host pointers, read during uhc_render_init only. */
typedef struct {
    int nshape, nplane;
    const double *plane;        /* [nshape][nplane][4] */
    const int *plane_adr;       /* [24] */
    const int *plane_num;       /* [24] */
    const double *sphere;       /* [nshape][24][4] */
} UhcRenderHulls;

/* MuJoCo's free camera (mjvCamera): eye = lookat - distance * (cos el cos az, cos el sin az, sin el), angles in degrees, fovy = vertical field
 * of view in degrees.  focus != 0 puts lookat x, y at each frame's root (the first humanoid's body 0).  shift_expert = x offset (m) of the
 * ghost; hide_im / hide_expert leave the first / the ghost humanoid out of the image (and out of the shadows). */
typedef struct {
    double lookat[3], azimuth, elevation, distance, fovy;
    int focus, hide_im, hide_expert;
    double shift_expert;
} UhcRenderCamera;

const char *uhc_render_last_error(void);   /* an alias of uhc_last_error (uhc_b200.h): the library keeps one error text */

/* Uploads the plane tables (as fp32) once per engine; a second call replaces them.  -2 unless nshape equals the engine's shape variants,
 * every body has 4 .. UHC_RENDER_MAX_PLANES planes inside 0 .. nplane - 1, and every value is finite.  Synchronises the device. */
int uhc_render_init(UhcEngine *e, const UhcRenderHulls *hulls);
/* Frees what uhc_render_init, uhc_render_mesh_init and their scratch hold (also safe without them); optional: uhc_engine_destroy frees it too. */
void uhc_render_release(UhcEngine *e);

/* The pose table [n][2][24][UHC_RENDER_POSE] fp32 of n frames: humanoid 0 = qpos row i, humanoid 1 = ghost row i (left untouched without a
 * ghost).  Rows are fp32 (precision 32) or fp64 (64), 76 values at qpos_dev + i * pitch (pitch >= 76: 148 reads the evaluation's state
 * record, 223 the tracker's state_out); the FK (motion_core.h) runs in fp64 with the frame's shape variant (variant_dev_or_null = [n],
 * NULL: 0), and only its result is rounded to fp32.  A variant array is copied to the host and range-checked, which synchronises `stream`. */
int uhc_render_pose(UhcEngine *e, long n, const void *qpos_dev, int precision, long pitch, const void *ghost_qpos_dev_or_null, long ghost_pitch,
                    const int *variant_dev_or_null, float *pose_dev, void *stream);
/* n frames of W x H pixels from a pose table [n][2][24][UHC_RENDER_POSE] (humanoids = 1: the ghost half is not read).  Outputs: rgb_dev =
 * [n][H][W][3] uint8; depth = [n][H][W] fp32 distance along the ray (m), +inf on sky; label = [n][H][W] uint8: 0 sky, 1 floor, 2 + b body b of
 * the first humanoid, 26 + b body b of the ghost.  Bad arguments (-2): no uhc_render_init, n < 0, W or H outside 1 .. 16384, humanoids not
 * 1 | 2, a null pose or rgb with n > 0, a camera with distance <= 0, fovy outside (0, 180) or a non-finite value, a variant out of range. */
int uhc_render_bodies(UhcEngine *e, const UhcRenderCamera *cam, int W, int H, long n, const float *pose_dev, int humanoids,
                      const int *variant_dev_or_null, unsigned char *rgb_dev, float *depth_dev_or_null, unsigned char *label_dev_or_null, void *stream);
/* uhc_render_pose into the engine's scratch, then uhc_render_bodies on it (the ghost present iff ghost_qpos_dev_or_null != NULL). */
int uhc_render_qpos(UhcEngine *e, const UhcRenderCamera *cam, int W, int H, long n, const void *qpos_dev, int precision, long pitch,
                    const void *ghost_qpos_dev_or_null, long ghost_pitch, const int *variant_dev_or_null, unsigned char *rgb_dev,
                    float *depth_dev_or_null, unsigned char *label_dev_or_null, void *stream);

/* ---- the skinned SMPL mesh (uhc_render_mesh): the same camera, floor, shading and outputs, with the posed mesh instead of the hulls.
 * The mesh is traced through a fixed two-level hierarchy, body -> leaves of at most UHC_RENDER_MESH_LEAF faces -> triangles, whose topology
 * uhc_b200/render_mesh.py builds once per model: face f belongs to the body whose SMPL joint has the largest summed skinning weight over its
 * three vertices, and every body's faces are split by a recursive median split of their rest-pose centroids.  Per frame only the boxes are
 * refitted. */
#define UHC_RENDER_MESH_LEAF 32

/* The topology, host pointers read during uhc_render_mesh_init only.  The faces are permuted so that leaf l holds faces leaf_first[l] ..
 * leaf_first[l + 1] - 1 and body b holds leaves body_leaf[b] .. body_leaf[b + 1] - 1 (leaves body-major); face_body[f] = the model body
 * (0 .. 23) of permuted face f. */
typedef struct {
    int nvert, nface, nleaf;
    const int *face;            /* [nface][3] vertex indices, 0 .. nvert - 1 */
    const int *face_body;       /* [nface] */
    const int *leaf_first;      /* [nleaf + 1] */
    const int *body_leaf;       /* [25] */
} UhcRenderMesh;

/* Uploads the topology once per engine; a second call replaces it, a failed call leaves the previous one.  -2 with nothing uploaded unless
 * every index lies in 0 .. nvert - 1, every face lies in exactly one leaf and that leaf belongs to the face's body, every leaf holds 1 ..
 * UHC_RENDER_MESH_LEAF faces, every body's leaves are one contiguous range, and the leaf boxes of two humanoids fit the trace kernel's
 * shared memory.  uhc_render_release frees it too.  Synchronises the device. */
int uhc_render_mesh_init(UhcEngine *e, const UhcRenderMesh *mesh);
/* n frames of W x H pixels of the mesh: verts_dev = [n][V][3] fp32 (uhc_smpl_mesh's vertices) of the grey humanoid, ghost_verts_dev_or_null
 * the same of the red one (shifted by shift_expert in x), root_dev_or_null = [n][3] fp32, the first humanoid's root, where a camera with focus
 * looks (required then).  Outputs, labels (2 + b / 26 + b: the body b a face belongs to) and the camera as uhc_render_bodies.  Shading is flat:
 * the face normal, turned towards the viewer, with one shadow ray towards the light.  Boxes are refitted into the engine's scratch, which
 * grows with n.  Bad arguments (-2): uhc_render_bodies' (but no uhc_render_init is needed), no uhc_render_mesh_init, nvert != the
 * topology's, a null verts with n > 0, a null root with focus on. */
int uhc_render_mesh(UhcEngine *e, const UhcRenderCamera *cam, int W, int H, long n, const float *verts_dev, const float *ghost_verts_dev_or_null,
                    const float *root_dev_or_null, int nvert, unsigned char *rgb_dev, float *depth_dev_or_null, unsigned char *label_dev_or_null,
                    void *stream);

#ifdef __cplusplus
}
#endif
#endif
