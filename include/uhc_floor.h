/* uhc_floor.h -- C ABI of the floor-contact measurements (part of libuhc_b200.so): where the body's surface is relative to the floor z = 0.
 *
 * Reference interfaces replaced: compute_penetration / compute_skate (uhc/smpllib/smpl_eval.py:125-149), which compute_metrics runs over SMPL
 * mesh vertices, and the minimum vertex height behind fix_height_smpl / fix_height_smpl_vanilla / fix_height
 * (uhc/data_process/process_amass_db.py:126-219).  Here the surface is the convex hulls of the 24 collision bodies, the surface the simulator
 * collides: one warp per frame places the bodies with the fp64 FK of uhc_load_motions, transforms every hull vertex and reduces in a fixed
 * order (uhc_b200/csrc/floor_core.h).  The hulls are coarser than the mesh, so the numbers compare between runs of this engine and between
 * simulated and reference motion, not with numbers published from mesh vertices.
 * Pointers suffixed _dev are CUDA device pointers, _host host pointers.  Returns 0 on success, -2 on a bad argument (nothing is launched and
 * the engine stays usable), -1 on a CUDA error (uhc_last_error()).
 */
#ifndef UHC_FLOOR_H
#define UHC_FLOOR_H
#include "uhc_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* per-frame columns: min_z (m, the lowest vertex), pen_mm (-mean(z | z < 0) * 1000, 0 with no vertex below), skate_mm (over the vertices with
 * z <= 0 in this and the previous frame the mean of |d xy| * 1000, 0 with none and on a row without a previous frame), float_mm
 * (max(min_z, 0) * 1000), n_below (the number of vertices with z < 0) */
#define UHC_FLOOR_NCOL 5
/* feet columns of uhc_motion_floor: z of L_Ankle, R_Ankle, L_Toe, R_Toe (m), the joints height rules are written against.  The reference's own
 * rules (and MotionSet.floor_audit, uhc_b200/motion_lib.py) read only the toes, SMPL joints 10 and 11; the ankles are there for callers whose
 * rule is about the ankle, which costs two stores per frame. */
#define UHC_FLOOR_NFEET 4

/* the hull vertices in fp64, as uhc_b200/model.py holds them (UhcModelHost's hull / hull_adr / hull_num; the engine keeps its own copy in
 * its precision for the collision) */
typedef struct {
    int nshape, nvert;
    const double *hull;                /* [nshape][nvert][3] body frame */
    const int *hull_adr, *hull_num;    /* [24] vertices of body b: hull_adr[b] .. hull_adr[b] + hull_num[b] - 1 */
} UhcFloorHulls;

const char *uhc_floor_last_error(void);   /* an alias of uhc_last_error (uhc_b200.h): the library keeps one error text */

/* copies the hulls to the device, before any call below (and before an evaluation with floor_host, uhc_eval.h).  Called again it replaces
 * them: evaluation graphs captured with the earlier copy are keyed on it and are not replayed.  A failed call leaves what was there.
 * -2: a null pointer, nshape other than the engine's shape variants, nvert < 1, bodies whose ranges do not tile 0 .. nvert - 1 in order */
int uhc_floor_init(UhcEngine *e, const UhcFloorHulls *h);
void uhc_floor_release(UhcEngine *e);     /* optional: uhc_engine_destroy frees it too */

/* n frames, frame i's qpos (76 values) at qpos_dev + i * qpos_pitch elements, fp32 (precision 32) or fp64 (64): a pitch of 223 reads the
 * tracker's state_out rows, 148 the evaluation's state record, 76 a plain qpos array.  variant_dev_or_null = [n] shape variant per frame
 * (NULL: variant 0); it is copied to the host and range-checked, which synchronises `stream`.  first_dev_or_null = [n], 1 = the row has no
 * previous frame (the first of a clip, or unrelated rows such as the envs of a tracker); NULL = rows 0 .. n-1 are one clip.  Row 0 never has
 * one.  Row i with a previous frame reads row i - 1 with row i's variant and recomputes its vertices, so nothing is carried between
 * launches.  out_dev = [n][UHC_FLOOR_NCOL].
 * Bad arguments (-2): n < 0, a null pointer (qpos or out with n > 0), qpos_pitch < 76, precision other than 32 | 64, a variant outside
 * 0 .. the engine's shape variants - 1, no hulls (uhc_floor_init). */
int uhc_floor_qpos(UhcEngine *e, const void *qpos_dev, int precision, long n, long qpos_pitch, const int *variant_dev_or_null,
                   const int *first_dev_or_null, double *out_dev, void *stream);

/* The same reduction over raw motion, before any table is built: the arguments of uhc_load_motions (nclips clips of clip_len_host frames,
 * rows_host = concatenated rows of UHC_MOTION_SMPL | UHC_MOTION_QPOS, fk_model_host = shape variant per clip or NULL, chunk_frames as there),
 * converted by the code uhc_load_motions runs and chunked through pinned staging buffers as it does.  out_dev = [sum(len)][UHC_FLOOR_NCOL]
 * (skate_mm of a clip's frame 0 is 0), feet_dev_or_null = [sum(len)][UHC_FLOOR_NFEET].  The loaded clip table is not touched.  Synchronises
 * the device.  Bad arguments (-2): those of uhc_load_motions except that a clip may be 1 frame long, a null out_dev, no hulls. */
int uhc_motion_floor(UhcEngine *e, int nclips, const int *clip_len_host, int kind, int pose_dim, const double *rows_host,
                     const int *fk_model_host, int chunk_frames, double *out_dev, double *feet_dev_or_null);

/* uhc_floor_qpos over the tracker's last state_out ([E][UHC_TRACK_OUT] in the engine's precision, include/uhc_track.h), env e with the shape
 * variant of its clip (the fk_model of uhc_track_begin) and no previous frame (the envs are unrelated rows, so skate_mm is 0): the clip models
 * were range-checked when they were set, so nothing is copied and nothing synchronises.  out_dev = [E][UHC_FLOOR_NCOL].  -2 unless a tracker
 * (uhc_track_begin) still owns the engine's clip table, and without hulls. */
int uhc_track_floor(UhcEngine *e, const void *state_out_dev, double *out_dev, void *stream);

#ifdef __cplusplus
}
#endif
#endif
