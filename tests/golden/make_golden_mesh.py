"""Generate tests/golden/mesh.npz by running THE REFERENCE'S OWN InstantNeuS.extract_fields and extract_color
(src/InstantNeuS.py:402-455) on the CPU: the whole field at res 33, a seeded sample of 4096 entries at res 70 (which the
reference splits into 64-point chunks) and the colours of 4096 float64 vertices (inside the bound, on its faces, outside
realtime_bound and outside the bound), on a trained_like net with a non-cubic bound and realtime_bound inside it.

Stand-ins for what the reference imports (make_golden.install_stubs): tinycudann -> the oracle.neus_oracle restatement
(hash grid with its autograd input gradient, MLP), mcubes and trimesh -> empty modules (neither method calls them).

Run:  python tests/golden/make_golden_mesh.py      (needs the reference source tree, see make_golden.REF)
"""
import os

import numpy as np
import torch

import make_golden as mg
from oracle import neus_oracle  # noqa: E402  (make_golden puts the repository on sys.path)

BOUND = [[-2.0, 1.5], [-1.2, 1.8], [-1.0, 2.2]]
RT_BOUND = [[-1.7, 1.3], [-1.0, 1.6], [-0.8, 2.0]]
WEIGHTS_SEED = 5


def main():
    mg.install_stubs()
    neus_mod = mg.ref_import("src.InstantNeuS")
    from goslam_b200 import synthetic
    metas, total_entries = neus_oracle.hashgrid_meta()
    offs = [m["offset"] * 2 for m in metas] + [total_entries * 2]
    ress = [m["res"] for m in metas]
    w = synthetic.make_neus_weights(seed=WEIGHTS_SEED, total_grid_params=total_entries * 2, layout=(offs, ress))
    net = neus_mod.InstantNeuS(synthetic.NEUS_CFG, BOUND, device="cpu")
    with torch.no_grad():
        net.sdf_network.encoding.encoding.params.copy_(w["grid"])
        net.sdf_network.sdf_layer.weight.copy_(w["sdf_w"])
        net.sdf_network.sdf_layer.bias.copy_(w["sdf_b"])
        net.color_network._B.copy_(w["color_B"])
        net.color_network.network.params.copy_(w["mlp"])
    net.update_bound(torch.tensor(RT_BOUND))
    u33 = net.extract_fields(net.bound[:, 0], net.bound[:, 1], 33)
    u70 = net.extract_fields(net.bound[:, 0], net.bound[:, 1], 70)
    g = np.random.default_rng(21)
    idx70 = np.sort(g.choice(70 ** 3, 4096, replace=False)).astype(np.int32)
    b = np.array(BOUND, np.float64)
    v = b[:, 0] + (b[:, 1] - b[:, 0]) * g.random((4096, 3))
    v[:512, 0] = np.where(g.random(512) < 0.5, b[0, 0], b[0, 1])              # on the x faces (normalised +-1)
    v[512:1024, 2] = np.where(g.random(512) < 0.5, b[2, 0], b[2, 1])          # on the z faces
    v[1024:1280] += g.normal(0.0, 0.3, (256, 3))                                # partly outside the bound (clamped)
    colors = net.extract_color(bound=net.bound.clone(), vertices=v)
    np.savez_compressed(os.path.join(mg.HERE, "mesh.npz"), bound=np.array(BOUND, np.float32),
                        rt_bound=np.array(RT_BOUND, np.float32), weights_seed=WEIGHTS_SEED, u33=u33,
                        idx70=idx70, u70=u70.reshape(-1)[idx70], vertices=v, colors=colors)


if __name__ == "__main__":
    if not os.path.isdir(mg.REF):
        raise SystemExit("needs the reference source tree (%s)" % mg.REF)
    main()
    print("wrote mesh")
