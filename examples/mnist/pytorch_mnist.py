#!/usr/bin/env python
"""MNIST with ``dear.DistributedOptimizer`` — the reference's example (examples/mnist/pytorch_mnist.py)
re-written for this framework.

    torchrun --nproc-per-node 2 examples/mnist/pytorch_mnist.py --epochs 1            # GPU(s), fused kernels
    DEAR_BACKEND=gloo torchrun --nproc-per-node 2 examples/mnist/pytorch_mnist.py --no-cuda   # CPU plumbing

There is no network in the build sandbox: if the MNIST files are not found under ``--data-dir`` a
deterministic synthetic MNIST-shaped dataset (class-dependent blobs, learnable) is used instead.
"""
from __future__ import annotations

import argparse
import os
import sys

import torch
import torch.nn.functional as F
import torch.utils.data
import torch.utils.data.distributed

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import dear_pytorch_b200 as hvd  # noqa: E402
from dear_pytorch_b200.models.mnist import Net  # noqa: E402


def synthetic_mnist(n: int, seed: int):
    g = torch.Generator().manual_seed(seed)
    y = torch.randint(0, 10, (n,), generator=g)
    protos = torch.randn(10, 1, 28, 28, generator=torch.Generator().manual_seed(7))
    x = 1.0 * protos[y] + 0.5 * torch.randn(n, 1, 28, 28, generator=g)
    return torch.utils.data.TensorDataset(x, y)


def load_datasets(data_dir: str, train_size: int, test_size: int):
    try:
        from torchvision import datasets, transforms
        tf = transforms.Compose([transforms.ToTensor(), transforms.Normalize((0.1307,), (0.3081,))])
        return (datasets.MNIST(data_dir, train=True, download=False, transform=tf),
                datasets.MNIST(data_dir, train=False, download=False, transform=tf))
    except Exception:
        return synthetic_mnist(train_size, 1), synthetic_mnist(test_size, 2)


def metric_average(val: float, name: str) -> float:
    t = torch.tensor([val], dtype=torch.float32, device=hvd.device())
    return float(hvd.allreduce(t, name=name).item())


def main(argv=None):
    ap = argparse.ArgumentParser(description="PyTorch MNIST Example (DeAR)")
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--test-batch-size", type=int, default=1000)
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--lr", type=float, default=0.01)
    ap.add_argument("--momentum", type=float, default=0.5)
    ap.add_argument("--no-cuda", action="store_true", default=False)
    ap.add_argument("--seed", type=int, default=42)
    ap.add_argument("--log-interval", type=int, default=10)
    ap.add_argument("--data-dir", default="./data")
    ap.add_argument("--train-size", type=int, default=6000)
    ap.add_argument("--test-size", type=int, default=1000)
    ap.add_argument("--threshold", type=float, default=0.05, help="fusion threshold in MB (the net has 0.08 MB)")
    ap.add_argument("--use-mixed-precision", action="store_true", default=False,
                    help="autocast forward + scaled loss (reference: train_mixed_precision, pytorch_mnist.py:63-83)")
    ap.add_argument("--loss-scale", type=float, default=None,
                    help="static loss scale of the mixed-precision path (default: dynamic, dear.GradScaler)")
    # parsed by the reference's example too, where only --use-adasum has an effect (the learning rate is then not scaled
    # by the number of ranks; the Horovod compression / Adasum / predivide arguments are commented out there,
    # examples/mnist/pytorch_mnist.py:207-235 of the reference)
    ap.add_argument("--fp16-allreduce", action="store_true", default=False, help="accepted for command-line parity (no effect)")
    ap.add_argument("--use-adasum", action="store_true", default=False, help="do not scale the learning rate by the world size")
    ap.add_argument("--gradient-predivide-factor", type=float, default=1.0, help="accepted for command-line parity (no effect)")
    args = ap.parse_args(argv)
    cuda = not args.no_cuda and torch.cuda.is_available()

    hvd.init(backend=None if cuda else os.environ.get("DEAR_BACKEND", "gloo"))
    torch.manual_seed(args.seed)
    device = hvd.device()

    train_ds, test_ds = load_datasets(args.data_dir, args.train_size, args.test_size)
    train_sampler = torch.utils.data.distributed.DistributedSampler(train_ds, num_replicas=hvd.size(), rank=hvd.rank())
    test_sampler = torch.utils.data.distributed.DistributedSampler(test_ds, num_replicas=hvd.size(), rank=hvd.rank())
    train_loader = torch.utils.data.DataLoader(train_ds, batch_size=args.batch_size, sampler=train_sampler)
    test_loader = torch.utils.data.DataLoader(test_ds, batch_size=args.test_batch_size, sampler=test_sampler)

    model = Net().to(device)
    # scale the learning rate by the number of workers, as the reference example does
    lr_scaler = 1 if args.use_adasum else hvd.size()
    optimizer = torch.optim.SGD(model.parameters(), lr=args.lr * lr_scaler, momentum=args.momentum)
    optimizer = hvd.DistributedOptimizer(optimizer, model=model, threshold=args.threshold, verbose=hvd.rank() == 0)
    hvd.broadcast_parameters(model.state_dict(), root_rank=0)

    def train(epoch):
        model.train()
        train_sampler.set_epoch(epoch)
        for batch_idx, (data, target) in enumerate(train_loader):
            data, target = data.to(device), target.to(device)
            optimizer.zero_grad()
            loss = F.nll_loss(model(data), target)
            loss.backward()
            optimizer.step()
            if batch_idx % args.log_interval == 0 and hvd.rank() == 0:
                print("Train Epoch: {} [{}/{} ({:.0f}%)]\tLoss: {:.6f}".format(
                    epoch, batch_idx * len(data), len(train_sampler), 100.0 * batch_idx / len(train_loader), loss.item()))

    scaler = hvd.GradScaler(optimizer) if (args.use_mixed_precision and args.loss_scale is None) else None

    def train_mixed_precision(epoch):
        """The reference's GradScaler loop (examples/mnist/pytorch_mnist.py:63-83): synchronize -> unscale ->
        ``with optimizer.skip_synchronize(): step``.  Here the gradients never surface as tensors (Kernel A consumes
        them during back-propagation), so the un-scaling is a factor of the reduce-scatter epilogue instead of a pass
        over the gradients.  dear.GradScaler (default) keeps the reference's call sequence and scales dynamically on
        the device; ``--loss-scale X`` runs a static scale (``set_loss_scale``)."""
        model.train()
        train_sampler.set_epoch(epoch)
        if scaler is None:
            optimizer.set_loss_scale(args.loss_scale)
        amp_dtype = torch.bfloat16 if (device.type == "cpu" or torch.cuda.is_bf16_supported()) else torch.float16
        for batch_idx, (data, target) in enumerate(train_loader):
            data, target = data.to(device), target.to(device)
            optimizer.zero_grad()
            with torch.autocast(device.type, dtype=amp_dtype):
                loss = F.nll_loss(model(data).float(), target)
            if scaler is not None:
                scaler.scale(loss).backward()
                optimizer.synchronize()
                scaler.unscale_(optimizer)
                with optimizer.skip_synchronize():
                    scaler.step(optimizer)
                scaler.update()
            else:
                (loss * args.loss_scale).backward()
                with optimizer.skip_synchronize():
                    optimizer.step()
            if batch_idx % args.log_interval == 0 and hvd.rank() == 0:
                print("Train Epoch: {} [{}/{} ({:.0f}%)]\tLoss: {:.6f}\tLoss Scale: {}".format(
                    epoch, batch_idx * len(data), len(train_sampler), 100.0 * batch_idx / len(train_loader), loss.item(),
                    scaler.get_scale() if scaler is not None else args.loss_scale))

    def test():
        model.eval()
        test_loss, test_acc = 0.0, 0.0
        with torch.no_grad():       # (the reference evaluates with grad enabled and re-applies the last update)
            for data, target in test_loader:
                data, target = data.to(device), target.to(device)
                out = model(data)
                test_loss += F.nll_loss(out, target, reduction="sum").item()
                test_acc += out.argmax(1).eq(target).float().sum().item()
        test_loss /= len(test_sampler)
        test_acc /= len(test_sampler)
        test_loss = metric_average(test_loss, "avg_loss")
        test_acc = metric_average(test_acc, "avg_accuracy")
        if hvd.rank() == 0:
            print("\nTest set: Average loss: {:.4f}, Accuracy: {:.2f}%\n".format(test_loss, 100.0 * test_acc))
        return test_loss, test_acc

    for epoch in range(1, args.epochs + 1):
        (train_mixed_precision if args.use_mixed_precision else train)(epoch)
    optimizer.synchronize()
    result = test()
    hvd.shutdown()
    return result


if __name__ == "__main__":
    main()
