// subject_glue.h -- internal interface of the subject body builder (subject.cu) to the tracker's run-time subjects (track.cu) and the
// engine that owns them (step_kernel.cu).  Not part of the C ABI.
#pragma once
#include <cuda_runtime.h>
#include "../../include/uhc_subject.h"

namespace uhc {
namespace subjx {

struct Builder;   // a basis and its base model's tables on the device: the inputs of k_subject (subject.cu)

// validates base (its variant 0 is read) and basis as uhc_subject_bodies does and uploads them to the current device.  0, -2 for a bad
// argument (uhc_err() names it, prefixed with `who`), -1 on a CUDA error
int builder_create(const UhcModelHost *base, const UhcSubjectBasis *basis, const char *who, Builder **out);
void builder_free(Builder *b);
bool has_gender(const Builder *b, int g);
int nvert(const Builder *b);
// k_subject over n rows, enqueued on st: betas [n][10] and gender [n] (checked by the caller) on the device -> body_f [n][24][20],
// hull [n][nvert][3] and bad [n] (0, or 1 + the last body whose map inverts it), all in device memory
cudaError_t launch(const Builder *b, int n, const double *betas, const int *gender, double *body_f, double *hull, int *bad, cudaStream_t st);

}  // namespace subjx
}  // namespace uhc
