"""Builds libuhc_b200.so (CUDA, sm_90a) in-tree.  nvcc cross-compiles without a GPU."""
import os
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "libuhc_b200.so")
SRCS = ["step_kernel.cu", "nn_kernels.cu", "mlp_wgmma.cu", "rollout.cu", "ppo_update.cu", "video.cu"]
# compiled on their own without multiply-add contraction: the motion library, the evaluation metrics, the curriculum weights and the tracker's
# streamed rows and the SMPL export restate numpy / scipy's fp64 arithmetic operation for operation; the renderer's pixel path and the floor
# measurements must give the bits of their host emulations; the SMPL mesh writes its fused multiply-adds as explicit intrinsics, so its vertices
# are the same bits in every kernel that computes them; the subject
# body builder's derived columns restate model.py's numpy arithmetic and must give the bits of its host emulation
NO_FMA_SRCS = ["motion_lib.cu", "eval.cu", "curriculum.cu", "track.cu", "export.cu", "render.cu", "render_mesh.cu", "floor.cu", "mesh.cu", "subject.cu"]
DEPS = ["errors.h", "sim_core.h", "env_step.h", "motion_core.h", "eval_core.h", "eval_glue.h", "graph_cache.h", "group_core.h", "curriculum_core.h", "track_core.h", "track_obs.h", "track_glue.h", "smpl_export_core.h", "render_core.h", "render_mesh_core.h", "floor_core.h", "video_core.h", "mesh_core.h", "subject_core.h", "subject_glue.h", "../../include/uhc_b200.h", "../../include/uhc_nn.h", "../../include/uhc_rollout.h", "../../include/uhc_ppo.h", "../../include/uhc_eval.h", "../../include/uhc_track.h", "../../include/uhc_export.h", "../../include/uhc_render.h", "../../include/uhc_floor.h", "../../include/uhc_video.h", "../../include/uhc_mesh.h", "../../include/uhc_subject.h"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "--use_fast_math=false",
              "-Xcompiler", "-fPIC", "-shared", "-Xptxas", "-v", "--expt-relaxed-constexpr"]


def build(force=False, verbose=False, so=SO, defines=()):
    """so: the library to write (default: the in-tree one the package loads); defines: extra preprocessor macros ("NAME" or "NAME=VALUE"),
    e.g. build(so="/tmp/x/libuhc_b200.so", defines=["UHC_PHASE_CLOCKS"]) for an instrumented variant beside the production library."""
    csrc = os.path.join(HERE, "csrc")
    srcs = [os.path.join(csrc, s) for s in SRCS]
    nofma = [os.path.join(csrc, s) for s in NO_FMA_SRCS]
    deps = srcs + nofma + [os.path.join(csrc, d) for d in DEPS] + [os.path.abspath(__file__)]
    extra = os.environ.get("UHC_NVCC_EXTRA", "").split() + ["-D" + d for d in defines]
    # the extra flags the library at `so` was built with live in a stamp beside it (no stamp: none), so a library built with other
    # defines or UHC_NVCC_EXTRA is never taken for an up-to-date one
    stamp = so + ".flags"
    built_with = open(stamp).read() if os.path.exists(stamp) else ""
    if (not force and built_with == " ".join(extra) and os.path.exists(so)
            and os.path.getmtime(so) >= max(os.path.getmtime(d) for d in deps if os.path.exists(d))):
        return so
    if os.path.exists(stamp):
        os.remove(stamp)
    flags = [f for f in NVCC_FLAGS if f != "--use_fast_math=false"] + extra
    with tempfile.TemporaryDirectory() as tmp:
        objs = []
        for s in nofma:
            o = os.path.join(tmp, os.path.basename(s) + ".o")
            cmd = ["nvcc"] + [f for f in flags if f != "-shared"] + ["-fmad=false", "-c", "-o", o, s]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if verbose or r.returncode:
                print(r.stdout[-6000:], r.stderr[-12000:])
            if r.returncode:
                raise RuntimeError("nvcc failed")
            objs.append(o)
        cmd = ["nvcc"] + flags + ["-o", so] + srcs + objs + ["-ldl"]
        r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode:
        print(r.stdout[-6000:], r.stderr[-12000:])
    if r.returncode:
        raise RuntimeError("nvcc failed")
    if extra:
        with open(stamp, "w") as f:
            f.write(" ".join(extra))
    return so


if __name__ == "__main__":
    build(force=True, verbose=True)
