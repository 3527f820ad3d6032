// track_glue.h -- internal interface of the tracker (track.cu) to the engine (step_kernel.cu).  Not part of the C ABI.
#pragma once
#include <cuda_runtime.h>
#include "../../include/uhc_b200.h"
#include "motion_core.h"

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

}  // namespace trackx
}  // namespace uhc
