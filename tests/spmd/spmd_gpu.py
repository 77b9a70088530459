"""GPU-only checks of the NVLink backend: every allreduce algorithm against a
plain fp32 PyTorch reference, misaligned / ragged tensors, big messages,
stream semantics, host-staging toggle, large point-to-point transfers."""
import os
import unittest

import torch

import mpi4torch_b200 as m4t
from common import DEVICE, comm

P, R = comm.size, comm.rank
CUDA = DEVICE.type == "cuda"
_C = m4t._C


def make(rank, n, dtype, seed=0):
    g = torch.Generator().manual_seed(1000 * seed + rank)
    if dtype.is_floating_point:
        return torch.randn(n, generator=g).to(dtype)
    return torch.randint(-50, 50, (n,), generator=g).to(dtype)


def reference_sum(n, dtype, seed=0):
    acc = torch.zeros(n, dtype=torch.float64)
    for p in range(P):
        acc += make(p, n, dtype, seed).double()
    return acc


@unittest.skipUnless(CUDA, "needs the CUDA backend")
class TestBackendBringUp(unittest.TestCase):
    def test_backend_is_native(self):
        self.assertTrue(m4t.cuda_backend_ready())
        if R == 0:
            print(f"[gpu] {comm.describe()} heap_mode={m4t.heap_mode()} nvls={m4t.has_nvls()}", flush=True)
        self.assertIn(m4t.heap_mode(), ("vmm+multicast", "vmm", "cudaIpc"))


@unittest.skipUnless(CUDA, "needs the CUDA backend")
class TestAllreduceAlgorithms(unittest.TestCase):
    sizes = [1, 7, 8, 255, 4096, 65537, 1 << 20, (1 << 22) + 3]

    def _run(self, algo, dtype, sizes):
        _C.set_tuning("force_algo", algo)
        try:
            for n in sizes:
                x = make(R, n, dtype).to(DEVICE)
                y = comm.Allreduce(x, m4t.MPI_SUM)
                ref = reference_sum(n, dtype)
                got = y.double().cpu()
                if dtype in (torch.float64, torch.int32, torch.int64):
                    ok = torch.allclose(got, ref, rtol=1e-12, atol=1e-9)
                elif dtype == torch.float32:
                    ok = torch.allclose(got, ref, rtol=1e-5, atol=1e-5)
                else:
                    ok = torch.allclose(got, ref, rtol=2 ** -6, atol=2 ** -5)
                self.assertTrue(ok, f"algo {algo} {dtype} n={n}: max err {(got - ref).abs().max().item()}")
                # all ranks must hold identical bits
                self.assertTrue(torch.equal(y, comm.Bcast_(y.clone(), 0)), f"algo {algo} {dtype} n={n} differs across ranks")
        finally:
            _C.set_tuning("force_algo", 0)

    def test_oneshot(self):
        for dt in (torch.float32, torch.bfloat16, torch.float64, torch.int32):
            self._run(1, dt, [n for n in self.sizes if n <= (1 << 20)])

    def test_twoshot(self):
        for dt in (torch.float32, torch.bfloat16, torch.float16, torch.float64, torch.int64):
            self._run(2, dt, self.sizes)

    def test_nvls_or_auto(self):
        algo = 3 if m4t.has_nvls() else 0
        for dt in (torch.float32, torch.bfloat16, torch.float16):
            self._run(algo, dt, self.sizes)

    def test_min_max_16bit(self):
        for op, fn in ((m4t.MPI_MAX, torch.maximum), (m4t.MPI_MIN, torch.minimum)):
            for dt in (torch.bfloat16, torch.float16):
                n = 100_003
                x = make(R, n, dt).to(DEVICE)
                y = comm.Allreduce(x, op)
                ref = make(0, n, dt)
                for p in range(1, P):
                    ref = fn(ref, make(p, n, dt))
                self.assertTrue(torch.equal(y.cpu(), ref))

    def test_misaligned_views(self):
        base = make(R, 10_007, torch.float32).to(DEVICE)
        x = base[3:]  # 12-byte offset: not 16-byte aligned
        y = comm.Allreduce(x, m4t.MPI_SUM)
        ref = reference_sum(10_007, torch.float32)[3:]
        self.assertTrue(torch.allclose(y.double().cpu(), ref, rtol=1e-5, atol=1e-5))

    def test_fused_scale_accumulate_bf16(self):
        n = 300_001
        x = make(R, n, torch.bfloat16).to(DEVICE)
        acc = make(R, n, torch.bfloat16, seed=5).to(DEVICE)
        y = comm.AllreduceFused(x, m4t.MPI_SUM, 1.0 / P, acc)
        ref = reference_sum(n, torch.bfloat16) / P + make(R, n, torch.bfloat16, seed=5).double()
        self.assertTrue(torch.allclose(y.double().cpu(), ref, rtol=2 ** -6, atol=2 ** -5))

    def test_accumulate_epilogue_large_and_in_place(self):
        # two-shot / NVLS kernels at every world size (the one-shot path ends at 2 MiB x (P-1))
        for dt, n in ((torch.bfloat16, 4 * 1024 * 1024 + 3), (torch.float32, 3 * 1024 * 1024 + 1)):
            x = make(R, n, dt, seed=2).to(DEVICE)
            acc = make(R, n, dt, seed=7).to(DEVICE)
            y = comm.AllreduceFused(x, m4t.MPI_SUM, 0.5, acc)
            ref = 0.5 * reference_sum(n, dt, seed=2) + make(R, n, dt, seed=7).double()
            tol = dict(rtol=2 ** -6, atol=2 ** -4) if dt == torch.bfloat16 else dict(rtol=1e-5, atol=1e-4)
            self.assertTrue(torch.allclose(y.double().cpu(), ref, **tol), str(dt))
            # in place: param += scale * Allreduce(grad), accumulate operand == output
            p = acc.clone()
            torch.ops.mpi4torch_b200.allreduce_axpy_(p, x, 0.5)
            self.assertTrue(torch.allclose(p.double().cpu(), ref, **tol), f"in-place epilogue ({dt})")

    def test_reduce_scatter_and_allgather_backward_large(self):
        rows = 3000 + R  # rank-dependent extents, several loop trips per thread
        total = sum(3000 + p for p in range(P))
        for dt in (torch.bfloat16, torch.float32, torch.float64):
            x = torch.full((total, 1024), float(R + 1), dtype=dt, device=DEVICE)
            y = comm.Reduce_scatter(x, m4t.MPI_SUM, 0, rows)
            self.assertEqual(list(y.shape), [rows, 1024])
            self.assertTrue(bool((y == P * (P + 1) / 2).all()), str(dt))
        a = torch.full((rows, 1024), 1.0, dtype=torch.float32, device=DEVICE, requires_grad=True)
        g = comm.Allgather(a, 0)
        self.assertEqual(g.shape[0], total)
        (g * float(R + 1)).sum().backward()  # adjoint = reduce-scatter of every rank's upstream gradient
        self.assertTrue(bool((a.grad == P * (P + 1) / 2).all()))

    def test_rooted_reduce_and_bcast_large(self):
        root = (P - 1) // 2
        for dt in (torch.bfloat16, torch.float32, torch.int32):
            n = 5 * 1024 * 1024 + 3
            x = torch.full((n,), R + 1, dtype=dt, device=DEVICE)
            y = comm.Reduce_(x, m4t.MPI_SUM, root)
            expect = P * (P + 1) // 2 if R == root else 0
            self.assertTrue(bool((y == expect).all()), f"Reduce_ {dt}")
            z = comm.Bcast_(torch.full((n,), R + 7, dtype=dt, device=DEVICE), root)
            self.assertTrue(bool((z == root + 7).all()), f"Bcast_ {dt}")

    def test_large_message(self):
        n = int(os.environ.get("M4T_TEST_BIG_ELEMS", str(32 * 1024 * 1024 + 5)))
        x = torch.full((n,), float(R + 1), dtype=torch.bfloat16, device=DEVICE)
        y = comm.Allreduce(x, m4t.MPI_SUM)
        self.assertTrue(bool((y == P * (P + 1) / 2).all()))

    def test_back_to_back_ops_reuse_staging_safely(self):
        outs = []
        for k in range(12):
            x = torch.full((50_000 + k,), float(R + k), dtype=torch.float32, device=DEVICE)
            outs.append((k, comm.Allreduce(x, m4t.MPI_SUM)))
        for k, y in outs:
            self.assertTrue(bool((y == P * k + P * (P - 1) / 2).all()), f"iteration {k}")

    def test_collectives_on_a_side_stream(self):
        s = torch.cuda.Stream()
        x = torch.full((1 << 18,), float(R), dtype=torch.float32, device=DEVICE)
        with torch.cuda.stream(s):
            y = comm.Allreduce(x, m4t.MPI_SUM)
        z = comm.Allreduce(x + 1, m4t.MPI_SUM)  # default stream, chained after the side stream
        s.synchronize()
        torch.cuda.synchronize()
        self.assertTrue(bool((y == P * (P - 1) / 2).all()))
        self.assertTrue(bool((z == P * (P - 1) / 2 + P).all()))


@unittest.skipUnless(CUDA, "needs the CUDA backend")
class TestHostStagingToggle(unittest.TestCase):
    def test_staged_path_gives_the_same_answer(self):
        x = make(R, 5000, torch.float32).to(DEVICE)
        a = comm.Allreduce(x, m4t.MPI_SUM)
        m4t.deactivate_cuda_aware_mpi_support()
        try:
            b = comm.Allreduce(x, m4t.MPI_SUM)
            self.assertEqual(b.device, x.device)
        finally:
            m4t.activate_nvlink_transport()
        self.assertTrue(torch.allclose(a, b, rtol=1e-5, atol=1e-5))


@unittest.skipUnless(CUDA, "needs the CUDA backend")
class TestLargeP2P(unittest.TestCase):
    def test_80mb_ring(self):
        n = 10_000_000  # the reference's message size (tests/test_nonblocking.py:9)
        right, left = (R + 1) % P, (R + P - 1) % P
        x = (torch.arange(n, dtype=torch.double, device=DEVICE) + R).requires_grad_()
        s = comm.Isend(x, right, 0)
        r = comm.Irecv(m4t.JoinDummies(torch.empty_like(x), [s.dummy]), left, 0)
        sent = comm.Wait(m4t.JoinDummiesHandle(s, [r.dummy]))
        got = comm.Wait(m4t.JoinDummiesHandle(r, [sent]))
        (got * R).sum().backward()
        self.assertTrue(torch.equal(got.detach(), torch.arange(n, dtype=torch.double, device=DEVICE) + left))
        self.assertTrue(torch.equal(x.grad, right * torch.ones_like(x)))


@unittest.skipUnless(CUDA, "needs the CUDA backend")
class TestFusedAllreduceLinear(unittest.TestCase):
    def _weights(self, n, k):
        return [torch.randn(n, k, generator=torch.Generator().manual_seed(50 + p)).to(torch.bfloat16) for p in range(P)]

    def test_forward_matches_unfused_reference(self):
        from mpi4torch_b200.ops import allreduce_linear, has_fused_kernel

        n, k, m = 512, 256, 384
        ws = self._weights(n, k)
        x = torch.randn(m, k, generator=torch.Generator().manual_seed(9)).to(torch.bfloat16).to(DEVICE)
        w = ws[R].to(DEVICE).requires_grad_()
        w_avg = (sum(t.float() for t in ws) / P)
        ref = x.float().cpu() @ w_avg.t()
        for rep in range(3):  # parity of the W_avg double buffer
            y = allreduce_linear(x, w, comm)
            err = (y.float().cpu() - ref).abs().max().item()
            self.assertLess(err / (ref.abs().max().item() + 1e-6), 3e-2, f"rep {rep}")
        if R == 0:
            fused = has_fused_kernel() and P > 1 and m4t.has_nvls()
            print(f"[gpu] allreduce_linear fused path active: {fused}", flush=True)

    def test_backward_matches_composition(self):
        from mpi4torch_b200.ops import allreduce_linear

        n, k, m = 256, 128, 128
        ws = self._weights(n, k)
        x = torch.randn(m, k, generator=torch.Generator().manual_seed(3 + R)).to(torch.bfloat16).to(DEVICE)
        w1 = ws[R].to(DEVICE).requires_grad_()
        w2 = ws[R].to(DEVICE).requires_grad_()
        allreduce_linear(x, w1, comm).float().square().sum().backward()
        allreduce_linear(x, w2, comm, force_unfused=True).float().square().sum().backward()
        scale = w2.grad.float().abs().max().item() + 1e-6
        self.assertLess((w1.grad.float() - w2.grad.float()).abs().max().item() / scale, 5e-2)

    def test_wgmma_gemm_inside_spmd(self):
        x = torch.randn(300, 192, generator=torch.Generator().manual_seed(1)).to(torch.bfloat16).to(DEVICE)
        w = torch.randn(520, 192, generator=torch.Generator().manual_seed(2)).to(torch.bfloat16).to(DEVICE)
        y = torch.ops.mpi4torch_b200.gemm_bf16_tn(x, w)
        ref = x.float() @ w.float().t()
        self.assertLess((y.float() - ref).abs().max().item() / ref.abs().max().item(), 2e-2)


@unittest.skipUnless(CUDA, "needs the CUDA backend")
class TestFusedTrainingStep(unittest.TestCase):
    def _reference_step(self, w, x, t, lr):
        """The same step written with plain fp32 torch ops + the library's differentiable Allreduce."""
        w = w.detach().float().requires_grad_()
        w_avg = comm.Allreduce(w, m4t.MPI_SUM) / P
        y = x.float() @ w_avg.to(torch.bfloat16).float().t()
        local = (y - t.float()).square().sum() / (x.shape[0] * P)
        loss = comm.Allreduce(local.reshape(1), m4t.MPI_SUM)
        loss.backward()
        return float(loss), (w.detach() - lr * w.grad)

    def test_autograd_step_matches_fp32_reference(self):
        """loss.backward() through dp_linear_mse + Allreduce: every configuration of the model (optimizer
        inside the backward kernel or not, fused forward or not) against the fp32 composition."""
        from mpi4torch_b200.models import DPLinearModel

        for in_bwd, fused, rep in ((True, True, False), (True, True, True), (False, True, False), (False, False, False)):
            model = DPLinearModel(256, 512, comm, device=DEVICE, dtype=torch.bfloat16, lr=1e-2, seed=3, fused=fused,
                                  sgd_in_backward=in_bwd, assume_replicated=rep)
            g = torch.Generator().manual_seed(77 + R)
            for step in range(3):
                x = torch.randn(384, 256, generator=g).to(torch.bfloat16).to(DEVICE)
                t = torch.randn(384, 512, generator=g).to(torch.bfloat16).to(DEVICE)
                ref_loss, ref_w = self._reference_step(model.weight, x, t, 1e-2)
                lf = float(model.train_step(x, t))
                self.assertLess(abs(lf - ref_loss) / (abs(ref_loss) + 1e-6), 1e-2, f"{in_bwd},{fused} step {step}")
                diff = (model.weight.detach().float() - ref_w).abs().max().item()
                self.assertLess(diff, 2e-2, f"{in_bwd},{fused} step {step}")
                self.assertIsNone(model.weight.grad)
            # all ranks hold bit-identical weights after the fused reduce-scatter + SGD + multicast
            self.assertTrue(torch.equal(model.weight.detach(), comm.Bcast_(model.weight.detach().clone(), 0)))

    def test_in_backward_optimizer_is_active_when_supported(self):
        from mpi4torch_b200.models import DPLinearModel
        from mpi4torch_b200.ops import in_backward_sgd_supported

        model = DPLinearModel(256, 512, comm, device=DEVICE, dtype=torch.bfloat16, lr=1e-2, seed=4)
        x = torch.randn(384, 256).to(torch.bfloat16).to(DEVICE)
        t = torch.randn(384, 512).to(torch.bfloat16).to(DEVICE)
        expect = P == 1 or m4t.has_nvls()
        self.assertEqual(in_backward_sgd_supported(x, model.weight, comm), expect)
        loss = model.loss(x, t)
        self.assertIn("MPIAllreduceSumBackward", loss.grad_fn.name())  # the loss Allreduce is a graph node
        w0 = model.weight.detach().clone()
        loss.backward()
        if expect:
            self.assertIsNone(model.weight.grad)           # the update happened inside backward
            self.assertFalse(torch.equal(w0, model.weight.detach()))
        else:
            self.assertIsNotNone(model.weight.grad)
        # a hand-made change of the weight invalidates the prefetched parameter average
        with torch.no_grad():
            model.weight.mul_(0.5)
        ref_loss, _ = self._reference_step(model.weight, x, t, 1e-2)
        l2 = float(model.train_step(x, t))
        self.assertLess(abs(l2 - ref_loss) / (abs(ref_loss) + 1e-6), 1e-2)

    def test_stacked_fused_layers_keep_their_saved_average(self):
        """Three equal-shape fused forwards before backward (advisor finding, round 1): the saved W_avg
        must survive the two-deep symmetric buffer being overwritten."""
        from mpi4torch_b200.ops import allreduce_linear

        n = k = 256
        ws = [torch.randn(n, k, generator=torch.Generator().manual_seed(60 + 7 * i + R)).to(torch.bfloat16).mul_(0.1)
              for i in range(3)]
        x = torch.randn(128, k, generator=torch.Generator().manual_seed(5 + R)).to(torch.bfloat16).to(DEVICE)
        outs = []
        for force in (False, True):
            xi = x.clone().requires_grad_()
            params = [w.to(DEVICE).requires_grad_() for w in ws]
            h = xi
            for p in params:
                h = allreduce_linear(h, p, comm, force_unfused=force)
            h.float().square().sum().backward()
            outs.append((xi.grad.float(), [p.grad.float() for p in params]))
        scale = outs[1][0].abs().max().item() + 1e-6
        self.assertLess((outs[0][0] - outs[1][0]).abs().max().item() / scale, 5e-2)
        for a, b in zip(outs[0][1], outs[1][1]):
            self.assertLess((a - b).abs().max().item() / (b.abs().max().item() + 1e-6), 5e-2)

    def test_fused_wgrad_update_matches_composition(self):
        if P < 2 or not m4t.has_nvls():
            return
        N, K, Mb = 512, 256, 384
        g = torch.Generator().manual_seed(5)
        w0 = (torch.randn(N, K, generator=g) * 0.1).to(torch.bfloat16)
        w = m4t.symmetric_empty((N, K), torch.bfloat16)
        w.copy_(w0)
        gr = torch.Generator().manual_seed(100 + R)
        gs = torch.full((1,), 2.0, device=DEVICE)
        for step in range(3):
            dy = torch.randn(Mb, N, generator=gr).to(torch.bfloat16).to(DEVICE)
            x = torch.randn(Mb, K, generator=gr).to(torch.bfloat16).to(DEVICE)
            ref_w = w.detach().clone()
            use_gs = step == 2
            gw = ((2.0 if use_gs else 1.0) * (dy.float().t() @ x.float())).to(torch.bfloat16)
            torch.ops.mpi4torch_b200.allreduce_axpy_(ref_w, gw, -0.01 / P)
            self.assertTrue(torch.ops.mpi4torch_b200.wgrad_allreduce_sgd_supported(w, dy, x))
            torch.ops.mpi4torch_b200.wgrad_allreduce_sgd_(w, dy, x, -0.01 / P, gs if use_gs else None)
            torch.cuda.synchronize()
            self.assertLess((w.float() - ref_w.float()).abs().max().item(), 2e-2, f"step {step}")
            self.assertTrue(torch.equal(w, comm.Bcast_(w.detach().clone(), 0)))
        # prefetch variant: also returns Allreduce(w_new) / P
        dy = torch.randn(Mb, N, generator=gr).to(torch.bfloat16).to(DEVICE)
        x = torch.randn(Mb, K, generator=gr).to(torch.bfloat16).to(DEVICE)
        w_avg = torch.ops.mpi4torch_b200.wgrad_allreduce_sgd_prefetch_(w, dy, x, -0.01 / P)
        torch.cuda.synchronize()
        expect = comm.AllreduceFused(w.detach().clone(), m4t.MPI_SUM, 1.0 / P, None)
        self.assertLess((w_avg.float() - expect.float()).abs().max().item(), 1e-2)
        if P & (P - 1) == 0:
            # replicated weights and a power-of-two world: the average of identical copies is exact, so a
            # stale read-back (the update not yet visible when the average was taken) cannot hide
            self.assertTrue(torch.equal(w_avg, w.detach()))
        # a second, large step: the prefetched average must follow the NEW weights
        w_before = w.detach().clone()
        w_avg2 = torch.ops.mpi4torch_b200.wgrad_allreduce_sgd_prefetch_(w, dy, x, -1.0 / P)
        torch.cuda.synchronize()
        self.assertGreater((w.float() - w_before.float()).abs().max().item(), 1.0)
        if P & (P - 1) == 0:
            self.assertTrue(torch.equal(w_avg2, w.detach()))
        else:
            self.assertLess((w_avg2.float() - w.float()).abs().max().item(), 2e-2 * w.float().abs().max().item())
        t = torch.randn(Mb, N, generator=gr).to(torch.bfloat16).to(DEVICE)
        dy2, loss2 = torch.ops.mpi4torch_b200.linear_mse_forward_local(x, w_avg, t, 1.0, 1.0)
        ref = (x.float() @ w_avg.float().t() - t.float())
        self.assertLess(abs(float(loss2) - float(ref.square().sum())) / float(ref.square().sum()), 2e-2)

    @unittest.skipUnless(os.environ.get("M4T_ZERO_COPY_IN", "0") == "1", "zero-copy symmetric inputs: set M4T_ZERO_COPY_IN=1")
    def test_zero_copy_symmetric_input(self):
        if P < 2:
            return
        for dt, n in ((torch.bfloat16, 3 * 1024 * 1024 + 8), (torch.float32, 1 << 20), (torch.float64, 70001)):
            x = m4t.symmetric_empty((n,), dt)
            src = make(R, n, dt, seed=9).to(DEVICE)
            x.copy_(src)
            y = comm.Allreduce(x, m4t.MPI_SUM)
            ref = comm.Allreduce(src, m4t.MPI_SUM)  # staged path, same kernels otherwise
            self.assertTrue(torch.equal(y, ref), str(dt))
            self.assertTrue(torch.equal(x, src), "input must be untouched")

    def test_graphed_step_matches_eager_step(self):
        from mpi4torch_b200.models import DPLinearModel

        # prefetch=False: the captured step re-averages the weights itself, so resetting them by hand below is visible
        eager = DPLinearModel(256, 512, comm, device=DEVICE, dtype=torch.bfloat16, lr=1e-2, seed=5, fused=False, prefetch=False)
        graphed = DPLinearModel(256, 512, comm, device=DEVICE, dtype=torch.bfloat16, lr=1e-2, seed=5, fused=False,
                                prefetch=False)
        g = torch.Generator().manual_seed(300 + R)
        x = torch.randn(384, 256, generator=g).to(torch.bfloat16).to(DEVICE)
        t = torch.randn(384, 512, generator=g).to(torch.bfloat16).to(DEVICE)
        w0 = graphed.weight.detach().clone()
        replay, sx, st, loss = graphed.make_graphed_step(x, t)
        with torch.no_grad():
            graphed.weight.copy_(w0)  # undo the warm-up / capture steps
        graphed.optimizer.invalidate()
        for step in range(3):
            xb = torch.randn(384, 256, generator=g).to(torch.bfloat16).to(DEVICE)
            tb = torch.randn(384, 512, generator=g).to(torch.bfloat16).to(DEVICE)
            le = float(eager.train_step(xb, tb))
            sx.copy_(xb)
            st.copy_(tb)
            replay()
            self.assertLess(abs(float(loss) - le) / (abs(le) + 1e-6), 1e-3, f"step {step}")
        self.assertLess((graphed.weight.float() - eager.weight.float()).abs().max().item(), 1e-3)

    def test_allreduce_axpy_in_place(self):
        p = torch.full((1000,), 2.0, dtype=torch.float32, device=DEVICE)
        gsrc = torch.full((1000,), float(R + 1), dtype=torch.float32, device=DEVICE)
        torch.ops.mpi4torch_b200.allreduce_axpy_(p, gsrc, -0.5)
        self.assertTrue(bool((p == 2.0 - 0.5 * P * (P + 1) / 2).all()))


if __name__ == "__main__":
    unittest.main()
