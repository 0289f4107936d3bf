"""torchrun --nproc-per-node 2 tools/run_sharded_ba.py : one factor graph sharded over 2+ GPUs
(edges by source frame, one NCCL all-reduce of the reduced camera system per iteration) must
reproduce single-GPU droid_backends.ba."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import measure  # noqa: E402
measure.require_cuda("run_sharded_ba.py")
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    if rank == 0:
        measure.emit({})
    from goslam_b200 import droid_backends, parallel, synthetic
    num_kf, ht, wd = 16, 40, 80
    sc, g = synthetic.make_scene(num_kf=num_kf, ht=ht, wd=wd, seed=9, rgbd=True, with_fmaps=False)
    coords = synthetic.true_reprojection(sc)
    tg, wg, eta = synthetic.make_update(sc, coords[0], g, noise=0.6)
    t0, t1, iters = 1, num_kf, 3
    kx = torch.unique(torch.cat([torch.arange(t0, t1), sc["ii"]]))
    eta_f = torch.zeros(num_kf, ht, wd)
    eta_f[kx] = eta
    D = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in sc.items()}
    tg, wg, eta, eta_f = tg.to(dev), wg.to(dev), eta.to(dev), eta_f.to(dev)
    # single-GPU reference on every rank
    p1, d1 = D["poses"].clone(), D["disps"].clone()
    droid_backends.ba(p1, d1, D["intrinsics"][0].contiguous(), D["disps_sens"], tg, wg, eta, D["ii"], D["jj"],
                      t0, t1, iters, 1e-4, 0.1, False)
    # sharded
    p2, d2 = D["poses"].clone(), D["disps"].clone()
    be = parallel.CudaBackend(p2, d2, D["intrinsics"][0].contiguous(), D["disps_sens"], t0, t1)
    torch.cuda.synchronize(); dist.barrier()
    t_sharded = measure.cuda_time(lambda: parallel.sharded_ba(be, d2, tg, wg, eta_f, D["ii"], D["jj"], iters, 1e-4, 0.1),
                                  1, warmup=0)["median_ms"]
    rel = lambda a, b: ((a - b).abs().max() / b.abs().max()).item()   # noqa: E731
    ok = rel(p2, p1) < 1e-5 and rel(d2, d1) < 1e-5
    print("rank %d/%d: poses rel %.2e disps rel %.2e  sharded BA %.1f us  %s" %
          (rank, world, rel(p2, p1), rel(d2, d1), 1e3 * t_sharded, "OK" if ok else "MISMATCH"), flush=True)
    # ---- the same through PEER MEMORY (goslam_ba_phase1_peers / goslam_ba_phase2_peers): no collective per iteration
    for (nk, h, w, lm, ep, its) in ((num_kf, ht, wd, 1e-4, 0.1, iters), (40, 30, 40, 1e-5, 1e-2, 2)):
        sc3, g3 = synthetic.make_scene(num_kf=nk, ht=h, wd=w, seed=11, rgbd=True, with_fmaps=False)
        tg3, wg3, eta3 = synthetic.make_update(sc3, synthetic.true_reprojection(sc3)[0], g3, noise=0.6)
        kx3 = torch.unique(torch.cat([torch.arange(1, nk), sc3["ii"]]))
        ef3 = torch.zeros(nk, h, w)
        ef3[kx3] = eta3
        E = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in sc3.items()}
        tg3, wg3, eta3, ef3 = tg3.to(dev), wg3.to(dev), eta3.to(dev), ef3.to(dev)
        pa, da = E["poses"].clone(), E["disps"].clone()
        droid_backends.ba(pa, da, E["intrinsics"][0].contiguous(), E["disps_sens"], tg3, wg3, eta3, E["ii"], E["jj"], 1, nk, its, lm, ep, False)
        pb = E["poses"].clone()
        n_sys = 36 * (nk - 1) ** 2 + 6 * (nk - 1)
        link = parallel.PeerLink(E["disps"], n_sys)
        be3 = parallel.PeerBackend(pb, link, E["intrinsics"][0].contiguous(), E["disps_sens"], 1, nk)
        bounds = parallel.shard_frames_by_edges(E["ii"], nk, world)
        lo, hi = bounds[rank]
        sel = parallel.local_edges(E["ii"], lo, hi)
        tl, wl, il, jl = tg3[sel].contiguous(), wg3[sel].contiguous(), E["ii"][sel].contiguous(), E["jj"][sel].contiguous()
        torch.cuda.synchronize(); dist.barrier()
        t_peer = measure.cuda_time(lambda: [be3.iteration(tl, wl, ef3, il, jl, lm, ep, False, lo, hi) for _ in range(its)],
                                   1, warmup=0)["median_ms"]
        link.wait_idle()
        torch.cuda.synchronize()
        db = link.disps.tensor
        ok3 = rel(pb, pa) < 1e-5 and rel(db, da) < 1e-5 and not bool(link.timeout.item())
        # every replica bit-identical: the partial systems are summed in rank order by every rank
        ref_p, ref_d = pb.clone(), db.clone()
        dist.broadcast(ref_p, src=0); dist.broadcast(ref_d, src=0)
        same = torch.equal(ref_p, pb) and torch.equal(ref_d, db)
        print("rank %d/%d: PEER exchange P=%d %dx%d: poses rel %.2e disps rel %.2e  %d iterations %.1f us  replicas identical %s  %s" %
              (rank, world, nk - 1, h, w, rel(pb, pa), rel(db, da), its, 1e3 * t_peer, same,
               "OK" if ok3 and same else "MISMATCH"), flush=True)
        ok = ok and ok3 and same
        link.close()
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
