"""The mesh renderer's static tables (include/uhc_render.h UhcRenderMesh), built once per SMPL model on the host.

The hierarchy has two fixed levels, body -> leaves -> triangles, and only its boxes change from frame to frame (the device refits them):
  - the body of a face is the SMPL joint with the largest summed skinning weight over the face's three vertices (ties: the lower joint),
    as the model body HumanoidModel.SMPL_BONE_ORDER maps it to, so labels mean what they mean for the hulls: 2 + 24 h + b;
  - every body's faces are split by a recursive median split of their rest-pose (v_template) centroids along the longest axis of the
    centroids' box, until a leaf holds at most LEAF faces;
  - leaves are stored body-major, and the faces are permuted so that every leaf is one contiguous run.
The build is deterministic: stable sorts and no random choice."""
import numpy as np

from .model import HumanoidModel

LEAF = 32          # include/uhc_render.h UHC_RENDER_MESH_LEAF


def face_bodies(faces, weights, body_names=None):
    """[F] model body of every face: the SMPL joint with the largest weight summed over its vertices (np.argmax: the lower joint on a tie)"""
    names = list(body_names or HumanoidModel().body_names)
    joint_body = np.array([names.index(n) for n in HumanoidModel.SMPL_BONE_ORDER], np.int32)
    w = np.asarray(weights, np.float64)
    f = np.asarray(faces, np.int64)
    return joint_body[np.argmax((w[f[:, 0]] + w[f[:, 1]]) + w[f[:, 2]], axis=1)]


def _split(idx, cen, out):
    if len(idx) <= LEAF:
        out.append(idx)
        return
    c = cen[idx]
    axis = int(np.argmax(c.max(0) - c.min(0)))                    # the first of equally long axes
    order = idx[np.argsort(c[:, axis], kind="stable")]
    half = len(order) // 2
    _split(order[:half], cen, out)
    _split(order[half:], cen, out)


def build_tables(faces, weights, v_template, body_names=None):
    """the topology uhc_render_mesh_init takes: dict(face [F][3] int32 (permuted), face_body [F] int32, leaf_first [L + 1] int32, body_leaf
    [25] int32, perm [F] int64: permuted face k is input face perm[k])"""
    faces = np.asarray(faces, np.int64)
    if faces.ndim != 2 or faces.shape[1] != 3 or len(faces) < 1:
        raise ValueError("render mesh: f (the faces) must be [F][3] with F >= 1")
    vt = np.asarray(v_template, np.float64)
    if faces.min() < 0 or faces.max() >= len(vt):
        raise ValueError(f"render mesh: f (the faces) holds a vertex index outside 0 .. {len(vt) - 1}")
    body = face_bodies(faces, weights, body_names)
    cen = vt[faces].mean(1)
    leaves, body_leaf = [], [0]
    for b in range(24):
        idx = np.nonzero(body == b)[0]
        if len(idx):                                               # a body that owns no face has no leaf
            _split(idx, cen, leaves)
        body_leaf.append(len(leaves))
    perm = np.concatenate(leaves)
    leaf_first = np.concatenate([[0], np.cumsum([len(x) for x in leaves])])
    return dict(face=np.ascontiguousarray(faces[perm], np.int32), face_body=np.ascontiguousarray(body[perm], np.int32),
                leaf_first=np.ascontiguousarray(leaf_first, np.int32), body_leaf=np.ascontiguousarray(body_leaf, np.int32), perm=perm)
