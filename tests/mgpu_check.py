"""Multi-GPU correctness on hardware (SURVEY.md section 4, "1-vs-2-vs-8 GPU equality"), run under torchrun on N GPUs of
one box (not collected by pytest; run it with torchrun on N = 2; bench.py's replica_check covers N = 8):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 tests/mgpu_check.py

  (1) FDS: every rank streams its rank::world shard of one feature matrix into the accumulators; after
      finish_epoch_stats (edge flags MAX-reduced, (count, sum, sum^2) SUM-reduced over NCCL) every rank's tables equal the
      oracle's statistics of the WHOLE matrix (rtol 1e-5) and are bit-identical across ranks;
  (2) gradients: the bucketed all-reduce that overlaps the backward pass gives exactly the buffer a single blocking
      all-reduce of the locally computed gradients gives (same NCCL sum), and equals the sum of the per-rank gradients
      gathered on every rank (rtol 1e-6: fp32 summation order);
  (3) one optimizer step later all replicas hold bit-identical parameters.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "imbalanced-regression_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    os.environ.setdefault("NCCL_DEBUG", "WARN")
    dist.init_process_group("nccl", device_id=dev)
    from oracle import dir_oracle as O
    from fds import FDS
    from resnet import ResNet, Bottleneck
    from parallel import DataParallel
    from optim import FusedAdam
    from loss import weighted_l1_loss

    # ---- (1) FDS statistics of a sharded epoch
    rng = np.random.RandomState(0)
    n, d, bn, bs = 5000, 256, 100, 3
    feats = np.maximum(rng.randn(n, d).astype(np.float32) * 0.7 + 1.0, 0)
    labels = rng.randint(0, 115, size=n).astype(np.float32)
    labels[labels == 3.0] = 4.0
    labels[0] = 3.0                     # the low edge value occurs in rank 0's shard only: the flag must be MAX-reduced
    m = FDS(d, bn, bs).to(dev)
    ref = O.FDSState(d, bn, bs)
    for ep in (0, 1):
        f, l = torch.from_numpy(feats).to(dev), torch.from_numpy(labels).to(dev)
        m.begin_epoch_stats(l[rank::world])
        m.accumulate_batch(f[rank::world], l[rank::world])
        m.update_last_epoch_stats(ep)
        m.finish_epoch_stats(ep)
        ref.update_last_epoch_stats(ep)
        ref.update_running_stats(feats, labels, ep)
        feats = feats * 1.05 + 0.01
    for k in ("running_mean", "running_var", "smoothed_mean_last_epoch", "num_samples_tracked"):
        got = getattr(m, k)
        np.testing.assert_allclose(got.cpu().numpy(), getattr(ref, k), rtol=1e-5, atol=1e-6, err_msg=k)
        other = got.clone()
        dist.broadcast(other, 0)
        assert torch.equal(other, got), f"FDS {k} differs between ranks"

    # ---- (2) gradients: overlapped buckets == one blocking all-reduce == sum of the local gradients
    torch.manual_seed(0)
    net = ResNet(Bottleneck, [2, 1, 1, 1], fds=True, bucket_num=100, bucket_start=3, start_update=0, start_smooth=1,
                 kernel="gaussian", ks=5, sigma=2, momentum=0.9).to(dev)
    model = DataParallel(net)
    model.broadcast_parameters()
    model.train()
    g = torch.Generator(device=dev).manual_seed(100 + rank)     # a different mini-batch on every rank
    x = torch.randn(16, 3, 64, 64, device=dev, generator=g)
    t = torch.randint(0, 100, (16, 1), device=dev, generator=g).float()
    w = torch.ones_like(t)

    def backward(hook):
        net._grad_bucket_hook = hook
        net.flat_grads().zero_()
        out, _ = model(x, t, 0)
        weighted_l1_loss(out, t, w).backward()

    backward(None)                                               # local gradients, nothing reduced yet
    local_g = net.flat_grads().clone()
    gathered = [torch.empty_like(local_g) for _ in range(world)]
    dist.all_gather(gathered, local_g)
    want = torch.stack(gathered).sum(0)
    blocking = local_g.clone()
    dist.all_reduce(blocking)
    backward(model._reduce_bucket)                               # overlapped: buckets go out during the backward pass
    assert len(model._works) == 4, len(model._works)            # layer4 .. layer1
    model.reduce_gradients()
    got = net.flat_grads()
    assert torch.equal(got, blocking), (got - blocking).abs().max().item()
    scale = want.abs().max().item()
    assert (got - want).abs().max().item() <= 1e-6 * scale, ((got - want).abs().max().item(), scale)

    # ---- (3) replicas stay bit-identical through the optimizer step
    opt = FusedAdam(model.parameters(), lr=1e-3, grad_scale=1.0 / world)
    opt.step()
    p = net.flat_parameters()
    p0 = p.clone()
    dist.broadcast(p0, 0)
    assert torch.equal(p, p0), "parameters differ between ranks after the step"
    dist.barrier()
    if rank == 0:
        print(f"mgpu_check ok: world {world}, FDS tables / bucketed gradients / parameters consistent", flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
