"""Generate tests/golden/mesh_eval.npz: the reconstruction evaluation (align_mesh / eval_mesh, src/mesher.py:339-421).

Inputs: the meshes oracle/mesh_oracle.py extracts from the mesh.npz scene at res 40 (the estimate) and res 48 (the
ground truth); the estimate's vertices moved by a known rigid motion P (1.5 degrees, 3 cm); seeded uniforms for
N3D samples of each mesh.

Outputs:
* the samples and face choices of oracle/mesh_eval_oracle.sample_surface for those uniforms;
* cKDTree nearest distances and indices both ways (gt samples -> est samples, est samples -> gt samples);
* the metrics and the message text of THE REFERENCE'S OWN eval_mesh, run on the CPU with stand-ins:
  trimesh.sample.sample_surface returns the oracle's samples for the stored uniforms, trimesh.PointCloud hands the
  vertices back, and the reference's cKDTree is scipy's (make_golden.install_stubs, empty open3d / pyrender /
  matplotlib modules);
* the ICP oracle's (T, fitness, rmse, iterations) for a rigid trans_init (P's inverse off by 0.5 degree and 1 cm) and
  for a scaled one (the same times a 1.01 scale), threshold 0.1.
No golden distance lies within 1e-12 of DIST_TH, so the threshold counts are well defined.

Run:  python tests/golden/make_golden_mesh_eval.py      (needs the reference source tree, see make_golden.REF)
"""
import contextlib
import io
import os
import sys
import tempfile
import types

import numpy as np

import make_golden as mg
from oracle import mesh_eval_oracle as meo  # noqa: E402  (make_golden puts the repository on sys.path)
from oracle import mesh_oracle, neus_oracle  # noqa: E402

RES_EST, RES_GT, N3D, DIST_TH, THRESHOLD, SEED = 40, 48, 4000, 0.05, 0.1, 17
PERTURB = meo.rigid([0.3, -0.5, 0.8], np.deg2rad(1.5), [0.03, -0.01, 0.02])


def meshes():
    from goslam_b200 import synthetic
    g = np.load(os.path.join(mg.HERE, "mesh.npz"))
    metas, tot = neus_oracle.hashgrid_meta()
    offs = [m["offset"] * 2 for m in metas] + [tot * 2]
    w = synthetic.make_neus_weights(seed=int(g["weights_seed"]), total_grid_params=tot * 2,
                                    layout=(offs, [m["res"] for m in metas]))
    _, ev, ef, _ = mesh_oracle.extract_mesh(w, g["bound"], g["rt_bound"], RES_EST, 0.0, color=False)
    _, gv, gf, _ = mesh_oracle.extract_mesh(w, g["bound"], g["rt_bound"], RES_GT, 0.0, color=False)
    return meo.transform(ev, PERTURB), ef, gv, gf


def reference_eval(est, gt, samples):
    """the reference's eval_mesh on stand-in meshes: (message, metrics file text)"""
    mg.install_stubs()
    tm = types.ModuleType("trimesh")
    tm.sample = types.SimpleNamespace(sample_surface=lambda mesh, count: samples[id(mesh)])
    tm.PointCloud = lambda vertices: types.SimpleNamespace(vertices=vertices)
    sys.modules["trimesh"] = tm
    for name in ("open3d", "pyrender", "matplotlib", "matplotlib.pyplot"):
        sys.modules[name] = types.ModuleType(name)
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    mesher = mg.ref_import("src.mesher")
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "metrics_mesh.txt")
        out = io.StringIO()
        with contextlib.redirect_stdout(out):
            mesher.eval_mesh(est, gt, N3d=N3D, dist_th=DIST_TH, out_path=path)
        text = open(path).read()
    assert out.getvalue() == text + "\n"
    return text


def main():
    ev, ef, gv, gf = meshes()
    rng = np.random.default_rng(SEED)
    u_est, u_gt = rng.random((N3D, 3)), rng.random((N3D, 3))
    s_est, f_est = meo.sample_surface(ev, ef, u_est)
    s_gt, f_gt = meo.sample_surface(gv, gf, u_gt)
    comp_d, comp_i = meo.nearest(s_gt, s_est)
    acc_d, acc_i = meo.nearest(s_est, s_gt)
    for d in (comp_d, acc_d):
        assert np.abs(d - DIST_TH).min() > 1e-12
    est = types.SimpleNamespace(vertices=ev, faces=ef)
    gt = types.SimpleNamespace(vertices=gv, faces=gf)
    msg = reference_eval(est, gt, {id(est): (s_est, f_est), id(gt): (s_gt, f_gt)})
    m = meo.metrics(s_est, s_gt, DIST_TH)
    inv = np.linalg.inv(PERTURB)
    inits = {"rigid": meo.rigid([1.0, 0.2, -0.4], np.deg2rad(0.5), [0.01, 0.0, -0.005]) @ inv}
    inits["scaled"] = np.diag([1.01, 1.01, 1.01, 1.0]) @ inits["rigid"]
    out = dict(est_verts=ev, est_faces=ef, gt_verts=gv, gt_faces=gf, perturb=PERTURB, u_est=u_est, u_gt=u_gt,
               s_est=s_est, f_est=f_est, s_gt=s_gt, f_gt=f_gt, comp_dist=comp_d, comp_idx=comp_i, acc_dist=acc_d,
               acc_idx=acc_i, message=np.array(msg), n3d=N3D, dist_th=DIST_TH, threshold=THRESHOLD,
               metrics=np.array([m[k] for k in ("accuracy", "completion", "accuracy_ratio", "completion_ratio",
                                                 "f_score")], np.float64))
    for name, init in inits.items():
        T, fit, rmse, it = meo.icp(ev, gv, THRESHOLD, init)
        out.update({"icp_init_" + name: init, "icp_T_" + name: T, "icp_fitness_" + name: fit,
                    "icp_rmse_" + name: rmse, "icp_iterations_" + name: it})
        print("%s: fitness %.6f rmse %.6f iterations %d" % (name, fit, rmse, it))
    np.savez_compressed(os.path.join(mg.HERE, "mesh_eval.npz"), **out)
    print("est V %d F %d, gt V %d F %d" % (len(ev), len(ef), len(gv), len(gf)) + msg)


if __name__ == "__main__":
    if not os.path.isdir(mg.REF):
        raise SystemExit("needs the reference source tree (%s)" % mg.REF)
    main()
    print("wrote mesh_eval")
