// track_glue.h -- internal interface of the tracker (track.cu) to the engine (step_kernel.cu).  Not part of the C ABI.
#pragma once
#include <cuda_runtime.h>
#include "../../include/uhc_b200.h"
#include "motion_core.h"
#include "subject_glue.h"

namespace uhc {
namespace trackx {

// null when the engine's cfg can run a stream of window H, else why not (obs v3, term_body root / Head, auto_reset, reactive_v 1, an `end`
// that could fire inside the window)
const char *cfg_error(const UhcEngine *e, int H);
// the clip table of the tracker: E clips x H rows (uninitialised), env records invalidated, clip models = fk_model (null: variant 0),
// shapes (null: zero) -- uhc_load_clips' table set-up.  fk_model must be in range (checked by the caller)
int install_table(UhcEngine *e, int H, const int *fk_model, const double *shape);
unsigned long long table_gen(const UhcEngine *e);
int num_shapes(const UhcEngine *e);
const motion::MotionModel &motion_model(const UhcEngine *e);
// the shape variant of every loaded clip on the device (uhc_set_clip_models, range-checked there); null while every clip uses variant 0
const int *clip_models(const UhcEngine *e);
// track.cu: a tracker (uhc_track_begin) owns the engine's current clip table, so env e follows clip e
bool tracking(UhcEngine *e);
// k_track_obs over every env into obs [E][obs_dim]; capturable
cudaError_t launch_obs(UhcEngine *e, float *obs, cudaStream_t st);

// ---- run-time subjects (uhc_track_subjects_enable / uhc_track_set_subjects)
// variant 0 of the engine's model in fp64: host arrays the engine keeps from its creation
UhcModelHost base_model(const UhcEngine *e);
// takes b (freeing an earlier builder).  The first call reserves slot nshape + env of body_f, hull and the FK body table for every env, as
// copies of variant 0, and the fp64 hull slots; the tables move, so the view generation changes and the rollout's graphs are dropped
int enable_subjects(UhcEngine *e, subjx::Builder *b);
const subjx::Builder *subject_builder(const UhcEngine *e);     // null until enable_subjects
// where uhc_track_set_subjects writes: body_f / hull [nshape + E][..] in the engine's precision, body6 [nshape + E][24][6] and hull64 [E][nvert][3]
// in fp64, the clip models (non-null while a tracker of an enabled engine owns the table), the shape rows and the env records
struct Slots {
    int nshape, nvert, precision;
    void *body_f, *hull; double *body6, *hull64;
    int *clip_model; void *shape; int *istate;
};
void slots(UhcEngine *e, Slots *s);
const double *slot_hulls(const UhcEngine *e);                  // [E][nvert][3] fp64, null until enabled

}  // namespace trackx
}  // namespace uhc
