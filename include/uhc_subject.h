/* uhc_subject.h -- C ABI of the subject body builder (part of libuhc_b200.so): humanoid shape variants from SMPL beta and gender.
 *
 * Reference interface replaced: HumanoidEnv.reset_robot (uhc/envs/humanoid_im.py:154-180), which rebuilds the MuJoCo humanoid from every
 * clip's beta and gender through Robot.load_from_skeleton (uhc/smpllib/smpl_robot.py:1018-1148).  This engine restates that body as the
 * shipped neutral humanoid carried onto the subject by one affine map per body, so that every variant keeps the shipped hull graph and can
 * be one of the engine's shape variants (UhcModelHost.nshape).  uhc_b200/subject_body.py fits the per-gender bases from the user's SMPL
 * files; this call evaluates them and everything that follows from them, in fp64, one CUDA block per subject (uhc_b200/csrc/subject_core.h
 * states the rules).  A row's outputs depend on its own beta and gender alone: they are the same bits alone or in any batch.
 * Needs no engine: call it before uhc_engine_create, whose UhcModelHost takes the variants it returns.
 */
#ifndef UHC_SUBJECT_H
#define UHC_SUBJECT_H
#include "uhc_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

#define UHC_SUBJECT_NBETA 10     /* shape components per subject (the reference trims the clip's 16 to 10 for smpl) */
#define UHC_SUBJECT_NTERM 11     /* basis terms: the constant, then one per shape component */

/* Per gender g (0 neutral, 1 male, 2 female; dataset_amass_single._gender_code), NULL where the gender has no model.  Indexed by model body
 * (uhc_b200/model.py order), z-up body frames:
 *   map[g]    [24][11][12]  (A | t) of the body's map as 3 rows of (A_i0, A_i1, A_i2, t_i): the constant term, then the 10 beta directions
 *   offset[g] [24][11][3]   the change of the body's offset from the shipped one: the constant term, then the 10 beta directions */
typedef struct {
    const double *map[3];
    const double *offset[3];
} UhcSubjectBasis;

/* n subjects: betas_host [n][10], gender_host [n].  Writes, per subject, the variant's body_f_host [n][24][20] and hull_host [n][nvert][3]
 * (UhcModelHost layouts; diffw and the pad column are copied from the base) and, when maps_host_or_null is not NULL, the 24 evaluated maps
 * [n][24][12].  `base` is the shipped model (its variant 0 is read).  Host pointers throughout; the call synchronises `device`.
 * Returns 0, -2 for a bad argument with nothing launched (a null pointer, n < 0, a gender outside 0 .. 2 or without a basis, a non-finite
 * beta) or, after the launch, for a subject with an inverted body (det A <= 0; nothing is written to the outputs), -1 on a CUDA error.
 * uhc_last_error() names the cause. */
int uhc_subject_bodies(int device, const UhcModelHost *base, const UhcSubjectBasis *basis, int n, const double *betas_host,
                       const int *gender_host, double *body_f_host, double *hull_host, double *maps_host_or_null);

#ifdef __cplusplus
}
#endif
#endif
