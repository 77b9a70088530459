"""Data-parallel MLP classifier (DPMLPClassifier: Linear -> GELU(tanh) -> Linear, softmax cross-entropy) on a
synthetic task: points drawn around one Gaussian centre per class.  Every rank draws its own batch; the parameters
stay identical on every rank, and each step prints the global loss and this step's accuracy over all ranks.

    python -m mpi4torch_b200.launch -np 2 examples/dp_mlp_classifier.py --device cpu
    python -m mpi4torch_b200.launch -np 8 examples/dp_mlp_classifier.py --features 1024 --hidden 4096 --classes 256

On CUDA the kernels need features, hidden and classes that are multiples of 128 and a batch that is a multiple
of 64; other shapes run the torch composition.
"""
import argparse

import torch

import mpi4torch_b200 as m4t
from mpi4torch_b200.models import DPMLPClassifier


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--features", type=int, default=128)
    ap.add_argument("--hidden", type=int, default=256)
    ap.add_argument("--classes", type=int, default=128)
    ap.add_argument("--lr", type=float, default=2.0)
    ap.add_argument("--device", default="cuda" if torch.cuda.is_available() else "cpu")
    args = ap.parse_args()
    comm = m4t.COMM_WORLD
    cuda = args.device == "cuda"
    device = torch.device("cuda", torch.cuda.current_device()) if cuda else torch.device("cpu")
    dtype = torch.bfloat16 if cuda else torch.float32
    model = DPMLPClassifier(args.features, args.hidden, args.classes, comm, device=device, dtype=dtype, lr=args.lr)
    centres = 2.0 * torch.randn(args.classes, args.features, generator=torch.Generator().manual_seed(7))
    g = torch.Generator().manual_seed(100 + comm.rank)  # every rank sees different data
    for step in range(args.steps):
        labels = torch.randint(0, args.classes, (args.batch,), generator=g)
        x = centres[labels] + torch.randn(args.batch, args.features, generator=g)
        x, labels = x.to(device, dtype), labels.to(device)
        correct = (model.logits(x).argmax(1) == labels).sum().to(torch.float64)
        loss = model.train_step(x, labels)
        accuracy = float(comm.Allreduce(correct, m4t.MPI_SUM)) / (args.batch * comm.size)
        if comm.rank == 0:
            print(f"step {step:3d}  loss {float(loss):.5f} accuracy {accuracy:.4f}", flush=True)


if __name__ == "__main__":
    main()
