"""Kernels and paths added between the rounds (3x3 weight gradient, stride-2 fprop through the TMA traversal stride,
stem kernel, column-loop BatchNorm-backward reduction in the dgrad epilogue, programmatic dependent launch, teacher
residual fusion, double-buffered feed, nvJPEG input path).  They run with the regular GPU suite."""
import os

import pytest
import torch

import f64_bounds as fb
from edl_b200 import ops

pytestmark = [pytest.mark.gpu]
DEV = "cuda"


def _rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


# the stem weight gradient (csrc/stem.cu) sums one fp32 partial per CTA: at most one CTA per SM
STEM_WGRAD_SPLIT = 132


WGRAD_SHAPES = [  # n, cin, cout, h, w      (ResNet50_vd stages first, then odd geometries)
    (8, 64, 64, 56, 56), (8, 128, 128, 28, 28), (8, 256, 256, 14, 14), (32, 512, 512, 7, 7),
    (2, 64, 128, 8, 16), (4, 128, 64, 14, 14), (3, 64, 192, 6, 8), (16, 64, 64, 7, 7), (2, 192, 64, 4, 28)]


@pytest.mark.parametrize("n,cin,cout,h,w", WGRAD_SHAPES)
@pytest.mark.parametrize("split", [1, 4, None])
def test_conv3x3_wgrad_repeatable(n, cin, cout, h, w, split):
    torch.manual_seed(0)
    x = torch.randn(n, cin, h, w, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    dy = (torch.randn(n, cout, h, w, device=DEV) * 0.1).bfloat16().contiguous(memory_format=torch.channels_last)
    wt = torch.zeros(cout, 3, 3, cin, device=DEV, dtype=torch.bfloat16)
    if not ops.conv3x3_wgrad_supported(x, wt):
        pytest.skip("geometry not supported by the pixel-box planner")
    k, sp = n * h * w, split if split is not None else ops.gemm.conv3x3_wgrad_split(n, h, w, cin, cout)
    got = ops.conv3x3_wgrad(x, dy, wt.shape, None, split_k=split)
    assert got.shape == wt.shape
    fb.check_bf16(got.view(cout, -1), *[t.reshape(cout, -1) for t in fb.wgrad_ref(x, dy, wt.shape)], k, sp,
                  what="conv3x3 wgrad")
    # accumulate into a sink (the flat gradient bucket): sink += dW, twice
    sink = torch.full((cout * 9 * cin,), 0.25, device=DEV, dtype=torch.bfloat16)
    want = fb.wgrad_ref(x, dy, wt.shape, sink=sink.clone())
    assert ops.conv3x3_wgrad(x, dy, wt.shape, sink, split_k=split) is None
    fb.check_bf16(sink.view(cout, -1), *[t.reshape(cout, -1) for t in want], k, sp, what="conv3x3 wgrad sink")
    # a second identical call gives the same bits, with and without a sink: no state carries over between calls
    assert torch.equal(ops.conv3x3_wgrad(x, dy, wt.shape, None, split_k=split), got)
    sink2 = torch.full_like(sink, 0.25)
    assert ops.conv3x3_wgrad(x, dy, wt.shape, sink2, split_k=split) is None
    assert torch.equal(sink2, sink)


def test_conv3x3_autograd_with_own_wgrad(monkeypatch):
    from edl_b200.ops import gemm as G

    monkeypatch.setattr(G, "OWN_WGRAD3", True)
    torch.manual_seed(1)
    x = torch.randn(4, 64, 28, 28, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    wt = (torch.randn(128, 3, 3, 64, device=DEV) * 0.05).bfloat16().requires_grad_(True)
    y = ops.conv3x3(x, wt)
    dy = torch.randn_like(y)
    y.backward(dy)
    xd, wd = x.detach(), wt.detach()
    fb.check_bf16(x.grad, *fb.dgrad_ref(dy, wd, x.shape), 9 * 128, what="conv3x3 dgrad")
    fb.check_bf16(wt.grad.view(128, -1), *[t.reshape(128, -1) for t in fb.wgrad_ref(xd, dy, wd.shape)], 4 * 28 * 28,
                  ops.gemm.conv3x3_wgrad_split(4, 28, 28, 64, 128), what="conv3x3 own wgrad")


def _chain(x, w1, w3, bn1, bn2, reps):
    """conv1x1 -> BN+ReLU -> conv3x3 -> BN, forward and backward, `reps` times (short dependent kernels)."""
    outs = []
    for _ in range(reps):
        xi = x.clone().requires_grad_(True)
        y = bn2(ops.conv3x3(bn1(ops.conv1x1(xi, w1)), w3))
        y.float().square().mean().backward()
        outs.append((y.detach().clone(), xi.grad.clone()))
    return outs


def test_programmatic_dependent_launch_matches_plain_launches():
    """EDL_PDL / set_pdl(True): the hot kernels start while their predecessor drains and must produce exactly the
    tensors of the fully serialised launches (eager and inside a captured CUDA graph)."""
    C = ops.native()
    torch.manual_seed(0)
    x = torch.randn(8, 64, 28, 28, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    w1 = (torch.randn(128, 64, device=DEV) * 0.1).bfloat16().requires_grad_(True)
    w3 = (torch.randn(128, 3, 3, 128, device=DEV) * 0.05).bfloat16().requires_grad_(True)
    bn1 = ops.BatchNormAct2d(128, relu=True).to(DEV).train()
    bn2 = ops.BatchNormAct2d(128, relu=False).to(DEV).train()
    assert not C.pdl_enabled()
    ref = _chain(x, w1, w3, bn1, bn2, 3)
    ref2 = _chain(x, w1, w3, bn1, bn2, 3)
    # BN statistics use float atomics: two plain runs already differ; that difference is the yardstick
    noise_y = max(_rel(a[0], b[0]) for a, b in zip(ref, ref2))
    noise_g = max(_rel(a[1], b[1]) for a, b in zip(ref, ref2))
    C.set_pdl(True)
    try:
        got = _chain(x, w1, w3, bn1, bn2, 3)
        torch.cuda.synchronize()
        for (y0, g0), (y1, g1) in zip(ref, got):
            assert _rel(y1, y0) < max(2e-3, 4 * noise_y), (_rel(y1, y0), noise_y)
            assert _rel(g1, g0) < max(2e-3, 4 * noise_g), (_rel(g1, g0), noise_g)
        # inside a graph: programmatic edges between consecutive kernel nodes (forward chain only: autograd's
        # gradient-accumulator nodes are pinned to the stream of the eager run above, see NOTES.md)
        def fwd():
            with torch.no_grad():
                return bn2(ops.conv3x3(bn1(ops.conv1x1(x, w1)), w3))

        bn1.eval(), bn2.eval()
        C.set_pdl(False)
        want = fwd()
        C.set_pdl(True)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            fwd()
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            cap = fwd()
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        assert torch.equal(cap, want)
    finally:
        C.set_pdl(False)


def test_step_pipelined_matches_step():
    """Double-buffered feed: same losses as the synchronous public step, handles readable one step late."""
    from edl_b200.models import ResNetVd, to_train_dtype
    from edl_b200.trainer import StudentTrainer

    def run(pipelined):
        torch.manual_seed(0)
        m = to_train_dtype(ResNetVd(18, class_dim=16, width_mult=0.25), torch.bfloat16, torch.device(DEV)).train()
        # a small learning rate: run-to-run float-atomic noise must not be amplified into different trajectories
        tr = StudentTrainer(m, 8, image_shape=(3, 32, 32), num_classes=16, lr=1e-3, use_graph=True)
        g = torch.Generator().manual_seed(1)
        xs = [torch.randn(8, 3, 32, 32, generator=g).bfloat16().contiguous(memory_format=torch.channels_last).pin_memory()
              for _ in range(3)]
        ts = [torch.softmax(torch.randn(8, 16, generator=g), -1).bfloat16().pin_memory() for _ in range(3)]
        losses, prev = [], None
        for i in range(9):
            if pipelined:
                h = tr.step_pipelined(xs[i % 3], ts[i % 3])
                if prev is not None:
                    losses.append(prev.item())
                prev = h
            else:
                losses.append(float(tr.step(xs[i % 3], ts[i % 3]).item()))
        if pipelined:
            losses.append(prev.item())
        return losses

    a, a2, b = run(False), run(False), run(True)
    assert len(a) == len(b) == 9
    noise = max(abs(u - v) for u, v in zip(a, a2))
    for u, v in zip(a, b):
        assert abs(u - v) <= max(2e-2 * max(1.0, abs(u)), 4 * noise), (a, a2, b)


def _agree_worker(rank, world, port, q):
    import torch.distributed as dist

    try:
        os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
        torch.cuda.set_device(rank)
        dev = torch.device("cuda", rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
        from edl_b200.models import ResNetVd, to_train_dtype
        from edl_b200.parallel import ElasticDataParallel

        m = to_train_dtype(ResNetVd(18, class_dim=16, width_mult=0.25), torch.bfloat16, dev)
        dp = ElasticDataParallel(m)
        assert dp.agree(0.0) == (0.0, 0)
        assert dp.agree(1.0 if rank == world - 1 else 0.0) == (1.0, 0)        # any rank's flag reaches every rank
        for _ in range(5):
            assert dp.agree(0.0) == (0.0, 0)
        if rank == 0:
            q.put("ok")
        dist.barrier()
        dist.destroy_process_group()
    except Exception as e:  # noqa: BLE001
        import traceback

        q.put("rank %d: %s\n%s" % (rank, e, traceback.format_exc()))
        raise


@pytest.mark.multigpu
def test_agreement_through_the_scalar_allgather_kernel():
    import torch.multiprocessing as mp

    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip("needs 2 GPUs")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29800 + os.getpid() % 1000
    procs = [ctx.Process(target=_agree_worker, args=(r, world, port, q)) for r in range(world)]
    [p.start() for p in procs]
    res = q.get(timeout=300)
    [p.join(60) for p in procs]
    assert res == "ok", res


def test_teacher_residual_fused_into_the_gemm_epilogue(monkeypatch):
    """EDL_TEACHER_FUSE_RES: relu(conv1x1 * scale + shift + residual) as one persistent-GEMM launch (scale folded into
    the weights, residual tile by TMA) against the two-kernel path and against fp32 math."""
    from edl_b200.models import resnext

    torch.manual_seed(0)
    conv = resnext.FoldedConv(256, 512, 1, relu=True).to(DEV)
    conv.weight.data = (torch.randn_like(conv.weight.float()) * 0.05).to(torch.bfloat16)
    conv.load_bn(torch.rand(512, device=DEV) + 0.5, torch.randn(512, device=DEV) * 0.1,
                 torch.randn(512, device=DEV) * 0.1, torch.rand(512, device=DEV) + 0.5)
    x = torch.randn(8, 256, 14, 14, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    res = torch.randn(8, 512, 14, 14, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    monkeypatch.setattr(resnext, "FUSE_RESIDUAL", False)
    two = conv(x, residual=res)
    monkeypatch.setattr(resnext, "FUSE_RESIDUAL", True)
    ops.reset_launches()
    one = conv(x, residual=res)
    assert ops.launches() == 1
    # the fused launch folds the scale into the weights: relu(x @ (w * scale) + shift + res), where w * scale is the bf16
    # weight the kernel reads; the two-kernel path applies scale and shift to the GEMM output, then adds the residual
    sc, sh = conv.scale.view(1, -1, 1, 1), conv.shift.view(1, -1, 1, 1)
    w = conv.weight.view(512, 1, 1, 256)
    fb.check_bf16(one, *fb.conv_ref(x, (w.float() * conv.scale.view(-1, 1, 1, 1)).bfloat16(), padding=0, add=res,
                                     shift=sh, relu=True), 256, what="teacher fused residual")
    # two kernels: the GEMM's bf16 output, then relu(y * scale + shift + residual) in fp32 on that output
    y1 = ops.gemm_bf16(fb.rows(x), w.view(512, 256))
    fb.check_bf16(y1, *fb.gemm_ref(fb.rows(x), w.view(512, 256)), 256, what="teacher gemm")
    y1 = y1.view(8, 14, 14, 512).permute(0, 3, 1, 2).double()
    two_ref = (torch.relu(y1 * sc + sh + res.double()), y1.abs() * sc.abs() + sh.abs() + res.double().abs())
    fb.check_bf16(two, *two_ref, 1, what="teacher scale_shift_act")
    # whole teacher: same logits either way
    m = resnext.to_inference_dtype(resnext.ResNeXt_tiny(), torch.bfloat16, DEV).eval()
    xi = torch.randn(4, 3, 64, 64, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    monkeypatch.setattr(resnext, "FUSE_RESIDUAL", False)
    a = m(xi).float()
    monkeypatch.setattr(resnext, "FUSE_RESIDUAL", True)
    b = m(xi).float()
    assert _rel(b, a) < 2e-2


def _hier_gpu_worker(rank, world, port, q):
    import torch.distributed as dist

    try:
        os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
        os.environ["EDL_FAKE_HOST"] = "node%d" % (rank // 2)              # 2 fake hosts x 2 GPUs on one box
        torch.cuda.set_device(rank)
        dev = torch.device("cuda", rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
        from edl_b200.models import ResNetVd, to_train_dtype
        from edl_b200.trainer import StudentTrainer

        torch.manual_seed(0)
        m = to_train_dtype(ResNetVd(18, class_dim=16, width_mult=0.25), torch.bfloat16, dev).train()
        for use_graph in (False, True):
            tr = StudentTrainer(m, 8, image_shape=(3, 32, 32), num_classes=16, lr=0.05, use_graph=use_graph, bucket_cap_mb=0.25)
            assert tr.dp.hier and tr.dp.local_world == 2 and tr.dp.use_symm
            torch.manual_seed(100 + rank)
            x = torch.randn(8, 3, 32, 32).bfloat16().contiguous(memory_format=torch.channels_last).pin_memory()
            t = torch.softmax(torch.randn(8, 16), -1).bfloat16().pin_memory()
            for _ in range(4):
                tr.step(x, t)
            torch.cuda.synchronize()
            flat = torch.cat([g.param.flatten().float() for g in tr.dp.flat.groups.values()])
            outs = [torch.empty_like(flat) for _ in range(world)]
            dist.all_gather(outs, flat)
            assert all(torch.equal(outs[0], o) for o in outs), "ranks diverged (graph=%s)" % use_graph
            assert torch.isfinite(flat).all() and tr.dp.check_comm_error() == 0
        if rank == 0:
            q.put("ok")
        dist.barrier()
        dist.destroy_process_group()
    except Exception as e:  # noqa: BLE001
        import traceback

        q.put("rank %d: %s\n%s" % (rank, e, traceback.format_exc()))
        raise


@pytest.mark.multigpu
def test_hierarchical_allreduce_on_fake_hosts():
    """Two-level gradient reduction (NVSwitch kernels inside a 'host', NCCL on 1/L slices across): 4 GPUs of one box
    pretending to be 2 hosts; replicas must stay bit-identical, eagerly and inside the step graph."""
    import torch.multiprocessing as mp

    world = 4
    if torch.cuda.device_count() < world:
        pytest.skip("needs 4 GPUs")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29850 + os.getpid() % 1000
    procs = [ctx.Process(target=_hier_gpu_worker, args=(r, world, port, q)) for r in range(world)]
    [p.start() for p in procs]
    res = q.get(timeout=400)
    [p.join(60) for p in procs]
    assert res == "ok", res


@pytest.mark.parametrize("n,cin,cout,h,w,groups", [(4, 128, 128, 56, 56, 1), (4, 256, 256, 28, 28, 1), (8, 512, 512, 14, 14, 1),
                                                   (2, 64, 128, 12, 20, 1), (2, 512, 512, 28, 28, 8), (2, 256, 256, 16, 16, 4)])
def test_conv3x3_stride2_fprop(n, cin, cout, h, w, groups):
    """3x3 / pad 1 / stride 2 forward on the persistent kernel (input sampled by the TMA traversal stride): training form
    with BN statistics, inference form with folded BN + ReLU, dense and grouped."""
    torch.manual_seed(0)
    x = torch.randn(n, cin, h, w, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    wt = (torch.randn(cout, 3, 3, cin // groups, device=DEV) * 0.05).bfloat16()
    if not ops.conv3x3_s2_supported(x, wt, groups):
        pytest.skip("shape not supported")
    ref = fb.conv_ref(x, wt, 2, 1, groups)
    scale = torch.rand(cout, device=DEV) + 0.5
    shift = torch.randn(cout, device=DEV) * 0.1
    y = ops.conv3x3_s2_infer(x, wt, scale, shift, True, groups)
    want = fb.conv_ref(x, wt, 2, 1, groups, scale=scale.view(1, -1, 1, 1), shift=shift.view(1, -1, 1, 1), relu=True)
    assert y.shape == want[0].shape
    fb.check_bf16(y, *want, 9 * cin // groups, what="conv3x3 s2 infer")
    if groups == 1:
        from edl_b200.ops import gemm as G

        # backward twice: library kernels (the default) and our own path (EDL_OWN_S2_BWD=1: zero-insertion + stride-1
        # wgmma dgrad, wgrad through the TMA traversal stride)
        for own in (False, True):
            prev, G.OWN_S2_BWD = G.OWN_S2_BWD, own
            try:
                stats = torch.zeros(2 * cout, device=DEV)
                xg = x.clone().requires_grad_(True)
                wg = wt.clone().requires_grad_(True)
                yt = ops.conv3x3_s2(xg, wg, stats)
                fb.check_bf16(yt, *ref, 9 * cin, what="conv3x3 s2")
                fb.check_sums(stats, *fb.stats_ref(yt), yt.numel() // cout, what="conv3x3 s2 stats")
                dy = torch.randn_like(yt)
                ops.reset_fallbacks()
                yt.backward(dy)
                assert bool(ops.fallbacks()) != own or not (G._s2_dgrad_supported(x, wt) and G._s2_wgrad_supported(x, wt))
                # own kernels or the library's: both pass the oracle (k of the weight gradient = output pixels,
                # split up to one per SM)
                fb.check_bf16(xg.grad, *fb.dgrad_ref(dy, wt, x.shape, 2), 9 * cout, what="conv3x3 s2 dgrad own=%s" % own)
                fb.check_bf16(wg.grad.view(cout, -1), *[t.reshape(cout, -1) for t in fb.wgrad_ref(x, dy, wt.shape, 2)],
                              dy.numel() // cout, 132, what="conv3x3 s2 wgrad own=%s" % own)
            finally:
                G.OWN_S2_BWD = prev


@pytest.mark.parametrize("m,k,n", [(2048, 64, 32), (5000, 64, 128), (6272, 512, 256), (300, 64, 1024), (100352, 64, 256)])
@pytest.mark.parametrize("relu,has_y", [(True, False), (True, True), (False, False)])
def test_bnr_mode2_gemm(m, k, n, relu, has_y):
    """Fused BatchNorm-backward reduction, column loop over the staged tiles: same contract as
    tests/test_persist_gpu.py, 1x1 dgrad epilogue."""
    torch.manual_seed(5)
    a = torch.randn(m, k, device=DEV).bfloat16()
    w = (torch.randn(k, n, device=DEV) * 0.1).bfloat16()
    x = torch.randn(m, n, device=DEV).bfloat16()
    y = torch.randn(m, n, device=DEV).bfloat16() if has_y else None
    h = fb.bn_hook(x, y, n, relu)
    d = ops.gemm_bf16(a, w, b_mn_major=True, bn=h)
    assert h.done
    fb.check_bf16(d, *fb.gemm_ref(a, w, b_mn_major=True), k, what="dgrad")
    fb.check_dsums(h, d, m, "dgrad dsums")


@pytest.mark.parametrize("nb,c,hh,ww", [(8, 64, 16, 16), (32, 256, 14, 14), (5, 64, 11, 20), (8, 256, 2, 2), (32, 64, 56, 56)])
def test_bnr_mode2_conv3x3(nb, c, hh, ww):
    torch.manual_seed(6)
    dy = torch.randn(nb, c, hh, ww, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    wt = (torch.randn(c, 3, 3, c, device=DEV) * 0.05).bfloat16()
    x = torch.randn(nb, c, hh, ww, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    h = fb.bn_hook(x, None, c, True)
    dx = torch.empty_like(x)
    ops.native().conv3x3(dy, wt, dx, True, None, h.as_list(nb * hh * ww, c), True)
    fb.check_bf16(dx, *fb.dgrad_ref(dy, wt, x.shape), 9 * c, what="conv3x3 dgrad")
    fb.check_dsums(h, dx, nb * hh * ww, "conv3x3 dgrad dsums")


@pytest.mark.parametrize("mode", [2])       # the only reduction mode; the parameter keeps the test ids stable
@pytest.mark.parametrize("m,k,n,with_add", [(100352, 64, 256, False), (100352, 64, 256, True), (25088, 512, 128, True),
                                            (6272, 1024, 2048, False),
                                            # M tails inside a tile, a partial N tile, 64-column tiles with the addend
                                            (50000, 128, 192, True), (7001, 256, 64, True), (33333, 64, 320, False),
                                            (129, 192, 512, True)])
def test_bnr_many_tiles_per_cta_and_addend(mode, m, k, n, with_add):
    """What the round-1 kernel tests did not cover and the model needs: several tiles per persistent CTA (x / y prefetch,
    barrier parities, constant reloads when the N tile changes) and the residual-gradient addend together with the
    BatchNorm reduction (every block's first 1x1 convolution)."""
    assert ops.native().get_bnr_mode() == mode
    torch.manual_seed(7)
    a = torch.randn(m, k, device=DEV).bfloat16()
    w = (torch.randn(k, n, device=DEV) * 0.05).bfloat16()
    x = torch.randn(m, n, device=DEV).bfloat16()
    y = torch.randn(m, n, device=DEV).bfloat16()
    add = torch.randn(m, n, device=DEV).bfloat16() if with_add else None
    h = fb.bn_hook(x, y, n, True)
    d = ops.gemm_bf16(a, w, b_mn_major=True, bn=h, add=add)
    assert h.done
    fb.check_bf16(d, *fb.gemm_ref(a, w, b_mn_major=True, add=add), k, what="dgrad")
    fb.check_dsums(h, d, m, "dgrad dsums")


@pytest.mark.parametrize("mode,batch", [pytest.param(2, 8, id="2"), pytest.param(2, 5, id="2-batch5")])
def test_fused_bn_backward_matches_unfused_at_model_level(monkeypatch, mode, batch):
    """EDL_FUSE_BN_BWD at model level: ResNet50_vd gradients with the BatchNorm reductions riding in the dgrad epilogues
    against the same model with the stand-alone reduction kernels; batch 5 leaves M tails in every layer."""
    import copy

    from edl_b200.models import ResNet50_vd, to_train_dtype
    from edl_b200.ops import gemm as G

    C = ops.native()
    torch.manual_seed(0)
    base = to_train_dtype(ResNet50_vd(class_dim=100), torch.bfloat16, torch.device(DEV)).train()
    x = torch.randn(batch, 3, 96, 96, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    t = torch.softmax(torch.randn(batch, 100, device=DEV), -1).bfloat16()

    def grads(fuse):
        m = copy.deepcopy(base)
        monkeypatch.setattr(G, "FUSE_BN_BWD", fuse)
        ops.reset_launches()
        loss = ops.soft_cross_entropy(m(x), t)
        loss.backward()
        torch.cuda.synchronize()
        return float(loss), ops.launches(), {n: p.grad.float().clone() for n, p in m.named_parameters()}

    assert C.get_bnr_mode() == mode
    l0, n0, g0 = grads(False)
    l0b, _, g0b = grads(False)          # run-to-run noise of the unfused path (float atomics in the BN statistics)
    l1, n1, g1 = grads(True)
    assert abs(l0 - l1) < max(1e-2, 4 * abs(l0 - l0b)), (l0, l0b, l1)
    assert n1 < n0 - 20, "the fused path should launch ~40 kernels fewer (%d vs %d)" % (n1, n0)
    noise = {k: _rel(g0b[k], g0[k]) for k in g0}
    bad = sorted(((_rel(g1[k], g0[k]), noise[k], k) for k in g0 if _rel(g1[k], g0[k]) > max(3e-2, 4 * noise[k])),
                 reverse=True)
    assert not bad, bad[:8]


@pytest.mark.parametrize("n,h,w", [(4, 224, 224), (3, 64, 96), (2, 33, 47), (2, 40, 56), (5, 18, 36)])
def test_stem_conv_direct_kernel(n, h, w):
    """EDL_OWN_STEM1: 3 -> 32 channel 3x3 / stride 2 stem convolution on the direct kernel with fused BN statistics."""
    torch.manual_seed(0)
    x = torch.randn(n, 3, h, w, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    wt = (torch.randn(32, 3, 3, 3, device=DEV) * 0.2).bfloat16().requires_grad_(True)
    stats = torch.zeros(64, device=DEV)
    y = ops.stem_conv(x, wt, stats)
    ref = fb.conv_ref(x, wt.detach(), 2, 1)
    assert y.shape == ref[0].shape and y.is_contiguous(memory_format=torch.channels_last)
    fb.check_bf16(y, *ref, 27, what="stem conv")
    fb.check_sums(stats, *fb.stats_ref(y), y.numel() // 32, what="stem conv stats")
    dy = torch.randn_like(y)
    y.backward(dy)
    fb.check_bf16(wt.grad.view(32, -1), *[t.reshape(32, -1) for t in fb.wgrad_ref(x, dy, wt.shape, 2)],
                  dy.numel() // 32, STEM_WGRAD_SPLIT, what="stem wgrad")


# ------------------------------------------------------------------ DALI-style input path (nvJPEG + fused augmentation)
def _jpeg_blobs(sizes, seed=0, quality=95):
    import cv2
    import numpy as np

    rng = np.random.RandomState(seed)
    blobs, imgs = [], []
    for h, w in sizes:
        img = cv2.GaussianBlur(rng.randint(0, 256, (h, w, 3)).astype(np.uint8), (9, 9), 0)
        ok, enc = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, quality])
        assert ok
        blobs.append(enc.tobytes())
        imgs.append(cv2.cvtColor(cv2.imdecode(enc, cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB))
    return blobs, imgs


def test_crop_resize_normalize_kernel_matches_the_numpy_model():
    import random

    import numpy as np

    from edl_b200.utils import image_pipeline as ip

    sizes = [(375, 500), (64, 48), (600, 401), (224, 224), (33, 1000)]
    rng = np.random.RandomState(1)
    imgs = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in sizes]
    aug = ip.GpuJpegAugmenter.__new__(ip.GpuJpegAugmenter)
    aug.size = 224
    for train in (True, False):
        items, total = aug.plan(sizes, random.Random(5), train)
        pool = torch.zeros(total, dtype=torch.uint8, device=DEV)
        for img, off in zip(imgs, items.view(np.int64)[:, 0]):
            pool[int(off):int(off) + img.size] = torch.from_numpy(img.reshape(-1)).to(DEV)
        y = torch.empty((len(sizes), 224, 224, 3), dtype=torch.bfloat16, device=DEV)
        ops.native().crop_resize_normalize(pool, torch.from_numpy(items).to(DEV), y, [0.485, 0.456, 0.406],
                                           [0.229, 0.224, 0.225])
        for i, img in enumerate(imgs):
            want = torch.from_numpy(ip.augment_reference(img, tuple(items[i, 3:7]), bool(items[i, 7]), 224))
            assert (y[i].float().cpu() - want).abs().max().item() < 0.03, (train, i)      # bf16 output rounding


@pytest.mark.parametrize("backend", ["default", "hardware"])
def test_nvjpeg_batched_decode_and_fused_augmentation(backend):
    import random

    import numpy as np

    from edl_b200.utils import image_pipeline as ip

    sizes = [(375, 500), (64, 48), (480, 640), (224, 224), (301, 203), (500, 333)]
    blobs, imgs = _jpeg_blobs(sizes)
    try:
        aug = ip.GpuJpegAugmenter(DEV, 224, backend=backend)
    except RuntimeError as e:
        if backend == "hardware":
            pytest.skip("no NVJPG engine backend: %s" % e)
        raise
    assert [(h, w) for h, w, _ in aug._dec.image_info(blobs)] == sizes
    x = aug(blobs, random.Random(11), train=True)
    torch.cuda.synchronize()
    assert x.shape == (6, 3, 224, 224) and x.dtype == torch.bfloat16 and bool(torch.isfinite(x.float()).all())
    items, _ = aug.plan(sizes, random.Random(11), True)               # same seed => same boxes
    for i, img in enumerate(imgs):
        # decoded pixels: IDCT / chroma upsampling differ slightly between libjpeg-turbo and nvJPEG
        off = int(items.view(np.int64)[i, 0])
        got = aug._pool[off:off + img.size].view(img.shape).cpu().numpy().astype(np.int32)
        assert np.abs(got - img.astype(np.int32)).mean() < 4.0, (i, np.abs(got - img.astype(np.int32)).mean())
        want = torch.from_numpy(ip.augment_reference(img, tuple(items[i, 3:7]), bool(items[i, 7]), 224))
        assert (x[i].permute(1, 2, 0).float().cpu() - want).abs().mean().item() < 0.05, i
    x1 = aug(blobs[:1], random.Random(11), train=False)               # single-image path + eval crop
    assert x1.shape == (1, 3, 224, 224)


@pytest.mark.parametrize("n,cout,h,w", [(4, 32, 112, 112), (2, 64, 112, 112), (3, 32, 20, 24)])
def test_32_channel_conv_in_pixel_pair_form(monkeypatch, n, cout, h, w):
    """EDL_OWN_STEM23: conv1_2 / conv1_3 of the stem (32 input channels) as a 64-channel convolution over pixel pairs:
    forward with fused BN statistics, input gradient and weight gradient against the fp32 reference."""
    from edl_b200.ops import gemm as G

    monkeypatch.setattr(G, "OWN_STEM23", True)
    torch.manual_seed(0)
    x = torch.randn(n, 32, h, w, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    wt = (torch.randn(cout, 3, 3, 32, device=DEV) * 0.1).bfloat16().requires_grad_(True)
    if not ops.conv3x3_pair_supported(x, wt):
        pytest.skip("geometry not supported")
    stats = torch.zeros(2 * cout, device=DEV)
    ops.reset_fallbacks()
    y = ops.conv3x3_pair(x, wt, stats)
    xd, wd = x.detach(), wt.detach()
    ref = fb.conv_ref(xd, wd)
    assert y.shape == ref[0].shape and y.is_contiguous(memory_format=torch.channels_last)
    fb.check_bf16(y, *ref, 9 * 64, what="pair conv")
    # the pair-form statistics are folded from 2 Cout channels: one more addition per channel
    fb.check_sums(stats, *fb.stats_ref(y), y.numel() // cout, what="pair conv stats")
    dy = torch.randn_like(y)
    y.backward(dy)
    fb.check_bf16(x.grad, *fb.dgrad_ref(dy, wd, x.shape), 9 * 2 * cout, what="pair dgrad")
    # pixel-pair weight gradient, then two of its bf16 taps folded into each of ours
    fb.check_pair_wgrad(wt.grad, xd, dy, wd.shape, n * h * w // 2,
                        ops.gemm.conv3x3_wgrad_split(n, h, w // 2, 64, 2 * cout) + 1)
    assert not ops.fallbacks(), ops.fallbacks()
