/* uhc_mesh.h -- C ABI of the SMPL body mesh (part of libuhc_b200.so): linear blend skinning of SMPL pose / translation on the device.
 *
 * Reference interfaces replaced: SMPL_Parser.get_joints_verts (uhc/smpllib/smpl_parser.py:335-360, smplx's SMPL forward and its lbs), which
 * HumanoidEnv.convert_2_smpl_params (uhc/envs/humanoid_im.py:127-150) runs under full_eval, and compute_penetration / compute_skate
 * (uhc/smpllib/smpl_eval.py:125-149) over the vertices it returns.  The model is the user's SMPL file (uhc_b200/smpl_model.py reads it); the
 * engine holds one upload of it.  Per row, in fp64: the axis-angles to rotations (smplx's batch_rodrigues), the pose feature and the 24-joint
 * chain (batch_rigid_transform).  Per vertex, in fp32 with fused multiply-adds in a fixed order: the 207-term pose blend, the skinning sum over
 * the joints of non-zero weight, then the translation added in fp64 and rounded once (uhc_b200/csrc/mesh_core.h).  A row's outputs depend on
 * its own pose, trans and shape (and, for the floor, its previous row) alone: they are the same bits wherever the row sits in a batch.
 * Pointers suffixed _dev are CUDA device pointers.  Returns 0 on success, -2 on a bad argument (nothing is launched and the engine stays
 * usable), -1 on a CUDA error (uhc_last_error()).  Calls on one engine share its scratch: issue them on one stream.
 */
#ifndef UHC_MESH_H
#define UHC_MESH_H
#include "uhc_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

#define UHC_SMPL_NJ 24        /* joints */
#define UHC_SMPL_NBETA 10     /* shape components (smplx's default num_betas) */
#define UHC_SMPL_NPOSE 207    /* pose-blend components: (R_k - I) of joints 1 .. 23, row-major */

/* an SMPL model in fp64, as uhc_b200/smpl_model.py load_smpl_model returns it */
typedef struct {
    int nvert;                    /* V */
    const double *v_template;     /* [V][3] */
    const double *shapedirs;      /* [V][3][10] */
    const double *posedirs;       /* [V][3][207] */
    const double *J_regressor;    /* [24][V] */
    const double *weights;        /* [V][24] */
    const int *parents;           /* [24], parents[0] = -1, 0 <= parents[k] < k */
} UhcSmplModel;

const char *uhc_mesh_last_error(void);   /* an alias of uhc_last_error (uhc_b200.h): the library keeps one error text */

/* copies the model to the device (skinning weights of exactly 0 are dropped: skipping a + 0 * A term is exact).  Called again it replaces
 * the model; a failed call leaves the previous one in place.  -2: a null pointer, nvert < 1, a parent table that is not a tree in order,
 * a non-finite value */
int uhc_mesh_init(UhcEngine *e, const UhcSmplModel *m);
void uhc_mesh_release(UhcEngine *e);     /* optional: uhc_engine_destroy frees it too */

/* n rows of SMPL pose_dev [n][72] (axis-angles of the 24 joints) and trans_dev [n][3] in fp64, exactly what uhc_qpos_to_smpl writes (so
 * qpos -> SMPL -> mesh stays on the device); betas_dev = [nbetas][10] shapes, row i takes betas_dev[beta_idx[i]] (beta_idx_dev_or_null
 * NULL: row 0).  The shape pass (v_template + shapedirs . beta and the rest joints J_regressor . v_shaped) runs once per row of betas_dev.
 * verts_dev_or_null = [n][V][3] fp32 (smplx's vertices + transl), joints_dev_or_null = [n][24][3] fp64 (smplx's joints[:, :24] + transl).
 * A beta_idx array is copied to the host and range-checked, which synchronises `stream`.
 * Bad arguments (-2): n < 0, nbetas < 1, a null pose, trans or betas with n > 0, no model (uhc_mesh_init), a beta_idx outside 0 .. nbetas - 1. */
int uhc_smpl_mesh(UhcEngine *e, long n, const double *pose_dev, const double *trans_dev, int nbetas, const double *betas_dev,
                  const int *beta_idx_dev_or_null, float *verts_dev_or_null, double *joints_dev_or_null, void *stream);

/* The mesh of the same rows against the floor z = 0, without writing a vertex to memory: out_dev = [n][UHC_FLOOR_NCOL] (include/uhc_floor.h:
 * min_z, pen_mm, skate_mm, float_mm, n_below) over the V vertices as uhc_smpl_mesh writes them, by the reference's rules: z < 0 is below the
 * floor, a vertex skates when z <= 0 in this row and the previous one.  Sums in fp64 in a fixed order.  first_dev_or_null = [n], 1 = the row
 * has no previous row (the first frame of a clip); NULL = rows 0 .. n-1 are one clip.  Row 0 never has one.  Inside a tile of consecutive
 * rows the previous row's vertices are reused; the first row of a tile recomputes its predecessor.
 * Bad arguments (-2): those of uhc_smpl_mesh, and a null out_dev with n > 0. */
int uhc_smpl_floor(UhcEngine *e, long n, const double *pose_dev, const double *trans_dev, int nbetas, const double *betas_dev,
                   const int *beta_idx_dev_or_null, const int *first_dev_or_null, double *out_dev, void *stream);

#ifdef __cplusplus
}
#endif
#endif
