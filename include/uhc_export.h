/* uhc_export.h -- C ABI of the SMPL export (part of libuhc_b200.so): simulated qpos back to SMPL pose / translation on the device.
 *
 * Reference interface replaced: qpos_to_smpl (uhc/smpllib/smpl_mujoco.py:738-752), which turns a [T][76] qpos array into an SMPL axis-angle
 * pose [T][24][3] (SMPL_BONE_ORDER_NAMES order) and a translation [T][3] through scipy's Rotation.  Here one thread per frame restates it in
 * fp64 (uhc_b200/csrc/smpl_export_core.h), the inverse of the SMPL -> qpos conversion of uhc_load_motions.
 * Pointers suffixed _dev are CUDA device pointers.  Returns 0 on success, -2 on a bad argument (nothing is launched and the engine stays
 * usable), -1 on a CUDA error (uhc_export_last_error()).
 */
#ifndef UHC_EXPORT_H
#define UHC_EXPORT_H
#include "uhc_b200.h"
#include "uhc_eval.h"   /* UHC_EVAL_SMPL: the 75 columns of one exported frame */
#ifdef __cplusplus
extern "C" {
#endif

const char *uhc_export_last_error(void);

/* n frames, frame i's qpos (76 values) at qpos_dev + i * qpos_pitch elements, fp32 (precision 32) or fp64 (64): a pitch of 223 reads the
 * tracker's state_out rows, 148 the evaluation's state record, 76 a plain qpos array.  variant_dev_or_null = [n] shape variant per frame
 * (NULL: variant 0); trans = qpos[0:3] minus that variant's root offset, so SMPL -> qpos (uhc_load_motions) -> SMPL round-trips for every
 * variant.  A variant array is copied to the host and range-checked, which synchronises `stream`.  pose_dev = [n][72], trans_dev = [n][3].
 * Bad arguments (-2): n < 0, a null pointer (qpos, pose or trans with n > 0), qpos_pitch < 76, precision other than 32 | 64, a variant
 * outside 0 .. the engine's shape variants - 1. */
int uhc_qpos_to_smpl(UhcEngine *e, const void *qpos_dev, int precision, long n, long qpos_pitch, const int *variant_dev_or_null,
                     double *pose_dev, double *trans_dev, void *stream);
/* The tracker's last state_out ([E][UHC_TRACK_OUT] in the engine's precision, include/uhc_track.h) as SMPL, env e with the shape variant of its
 * clip (the fk_model of uhc_track_begin): uhc_qpos_to_smpl at pitch 223 without the variant copy -- the clip models were range-checked when
 * they were set, so nothing synchronises.  -2 unless a tracker (uhc_track_begin) still owns the engine's clip table. */
int uhc_track_smpl(UhcEngine *e, const void *state_out_dev, double *pose_dev, double *trans_dev, void *stream);

#ifdef __cplusplus
}
#endif
#endif
