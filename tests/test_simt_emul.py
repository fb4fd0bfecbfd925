"""The persistent-MLP CUDA kernels (csrc/mlp_persistent.cu + mlp_v2.inc — the flagship op of BASELINE configs 1-3)
executed on the CPU: the kernel *source* is compiled with g++ through csrc/host_shim.h (one OS thread per CUDA thread,
__syncthreads / warp shuffles / dynamic shared memory emulated) and compared with the PyTorch definitions, exactly
like tests/test_gpu_kernels.py does on a GPU.  Every variant: v1 (weights in shared memory, 256 threads), v2 with 128
threads (register-resident row + column copies, replicated head) in its strided (3), blocked (5) and blocked + packed-FMA (6) forms."""
import pytest
import torch

from colearn_federated_learning_b200.models import build_model, flatten_params
from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.ops import reference

NETS = {  # kind: (model name, dims, output activation, losses)
    0: ("ffnn", (10, 50, 30, 10, 1), "sigmoid", ("bce", "sse", "mse")),
    1: ("mlp", (10, 64, 64, 2), "none", ("xent",)),
    2: ("testing_remote", (2, 50, 10, 1), "none", ("sse", "mse")),
}
LOSS_CODES = {"bce": 0, "sse": 1, "xent": 2, "mse": 3}


@pytest.fixture(scope="module")
def simt():
    import glob
    import importlib.util
    import os

    import shutil

    from colearn_federated_learning_b200.ops import build
    if shutil.which("g++") is None or not os.path.exists(os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include", "cuda_runtime.h")):
        pytest.skip("no g++ / CUDA headers on this box: the SIMT emulator cannot be built")
    path = build.build_simt_emul()          # a compile error in a kernel source is a test failure, not a skip
    spec = importlib.util.spec_from_file_location("_colearn_simt", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert glob.glob(os.path.join(os.path.dirname(path), "_colearn_simt*.so"))
    return mod


def _data(dims, loss, n, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, dims[0], generator=g)
    y = (torch.randint(0, dims[-1], (n, 1), generator=g).float() if loss == "xent"
         else (torch.rand(n, dims[-1], generator=g) > 0.5).float())
    return x, y


CASES = [(k, loss, v, b) for k, (_, _, _, losses) in NETS.items() for loss in losses for v, b in ((3, 1), (1, 1), (3, 4), (5, 1), (5, 4), (6, 1), (6, 4))]


@pytest.mark.parametrize("kind,loss,variant,batch", CASES)
def test_kernel_source_on_cpu_matches_reference(simt, kind, loss, variant, batch):
    name, dims, act, _ = NETS[kind]
    n = 23
    x, y = _data(dims, loss, n, seed=kind * 10 + batch)
    torch.manual_seed(kind)
    flat0 = flatten_params(build_model(name)).clone()
    assert simt.mlp_net_params(kind) == flat0.numel()
    perm = reference.make_permutation(n, 2, seed=5)
    want = flat0.clone()
    last = reference.mlp_local_sgd(want, dims, x, y, perm, batch, 0.05, 2, -1, loss, act)
    got = flat0.clone()
    losses = simt.mlp_local_sgd(kind, flat0, [got], [x], [y], [perm], batch, 2, -1, LOSS_CODES[loss], 0.05, variant, [1.0], False, None)
    torch.testing.assert_close(got, want, rtol=2e-3, atol=2e-4)
    assert abs(float(losses[0, 0]) - float(last)) < 2e-3 * max(1.0, abs(float(last)))


@pytest.mark.parametrize("kind", sorted(NETS))
@pytest.mark.parametrize("variant", [5, 6, 3, 1])
def test_in_kernel_shuffle_from_kernel_source(simt, kind, variant):
    """ClientDesc::perm_seed on the CPU shim: both gather forms (index ring with the bijection computed per sample for the
    4-layer net, kernel-made table in perm_scratch for the 3-layer nets, per-element in the smem-weights kernel) train through
    exactly the order feistel_perm_kernel tabulates for (seed, perm_row0 + epoch) — bit-identical parameters and losses."""
    name, dims, act, losses = NETS[kind]
    loss = losses[0]
    n, epochs, seed, row0 = 37, 3, 987654321, 5
    x, y = _data(dims, loss, n, seed=kind + 40)
    torch.manual_seed(kind)
    flat0 = flatten_params(build_model(name)).clone()
    table = simt.feistel_permutation(n, row0 + epochs, seed)
    a, b = flat0.clone(), flat0.clone()
    la = simt.mlp_local_sgd(kind, flat0, [a], [x], [y], [table[row0:].contiguous()], 1, epochs, -1, LOSS_CODES[loss], 0.05, variant, [1.0], False, None)
    scratch = torch.full((1, epochs * n), -1, dtype=torch.int32)
    lb = simt.mlp_local_sgd(kind, flat0, [b], [x], [y], [None], 1, epochs, -1, LOSS_CODES[loss], 0.05, variant, [1.0], False, None,
                            perm_seed=seed, perm_row0=row0, perm_scratch=scratch)
    assert torch.equal(a, b) and torch.equal(la, lb)
    assert not torch.equal(a, flat0)
    if variant != 1 and len(dims) - 1 < 4:                       # the table form leaves the order it used behind
        assert torch.equal(scratch.view(epochs, n), table[row0:])


def test_step_limit_scale_delta_flags_and_many_clients(simt):
    """max_nr_batches, the FedAvg weight pre-applied by the producer (out = w * theta_k or w * (theta_k - theta_in)), the
    completion flag (st.release) and one CTA per client — the star protocol's worker side."""
    kind, (name, dims, act, _) = 1, NETS[1]
    flat0 = flatten_params(build_model(name)).clone()
    k = 3
    xs, ys, perms, wants = [], [], [], []
    for i in range(k):
        x, y = _data(dims, "xent", 17 + i, seed=i)
        p = reference.make_permutation(17 + i, 1, seed=i)
        w = flat0.clone()
        reference.mlp_local_sgd(w, dims, x, y, p, 1, 0.1, 3, 11, "xent", act)       # 3 epochs, capped at 11 steps
        xs.append(x), ys.append(y), perms.append(p), wants.append(w)
    outs = [torch.zeros_like(flat0) for _ in range(k)]
    flags = torch.zeros(k, dtype=torch.int32)
    scales = [0.5, 0.25, 0.25]
    simt.mlp_local_sgd(kind, flat0, outs, xs, ys, perms, 1, 3, 11, LOSS_CODES["xent"], 0.1, 3, scales, False, flags)
    for i in range(k):
        torch.testing.assert_close(outs[i], scales[i] * wants[i], rtol=2e-3, atol=2e-4)
    assert flags.tolist() == [7, 8, 9]
    deltas = [torch.zeros_like(flat0) for _ in range(k)]
    simt.mlp_local_sgd(kind, flat0, deltas, xs, ys, perms, 1, 3, 11, LOSS_CODES["xent"], 0.1, 3, scales, True, None)
    for i in range(k):
        torch.testing.assert_close(deltas[i], scales[i] * (wants[i] - flat0), rtol=2e-3, atol=2e-4)
    # FedAvg of the pre-scaled contributions = the weighted mean of the locally trained models
    torch.testing.assert_close(sum(outs), sum(s * w for s, w in zip(scales, wants)), rtol=2e-3, atol=2e-4)


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_forward_kernel_on_cpu(simt, kind):
    name, dims, act, _ = NETS[kind]
    flat = flatten_params(build_model(name)).clone()
    x = torch.rand(41, dims[0])
    got = simt.mlp_forward(kind, flat, x, dims[-1])
    torch.testing.assert_close(got, reference.mlp_forward(flat, dims, x, act)[0], rtol=1e-4, atol=1e-5)


# ---- elementwise.cu on the CPU -------------------------------------------------------------------------------------------
def test_elementwise_kernels_on_cpu(simt):
    torch.manual_seed(0)
    n = 5000 + 3                                             # not a multiple of the vector width: scalar tails run too
    p, g = torch.randn(n), torch.randn(n)
    want = p - 0.05 * g
    simt.sgd_step(p, g, 0.05)
    torch.testing.assert_close(p, want, rtol=1e-6, atol=1e-6)
    k = 5
    slots, w, theta = torch.randn(k, n), torch.softmax(torch.randn(k), 0), torch.randn(n)
    torch.testing.assert_close(simt.fedavg_flat(slots, w), reference.fedavg_flat(slots, w), rtol=1e-5, atol=1e-5)
    want = reference.fedavg_apply(theta.clone(), slots, w, 0.7)
    simt.fedavg_apply(theta, slots, w, 0.7)
    torch.testing.assert_close(theta, want, rtol=1e-5, atol=1e-5)
    z, y = torch.randn(777) * 3, (torch.rand(777) > 0.5).float()
    loss, dz = simt.sigmoid_bce(z, y)
    rl, rdz = reference.sigmoid_bce(z, y)
    torch.testing.assert_close(loss, rl, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(dz, rdz, rtol=1e-4, atol=1e-6)
    out, yy = torch.randn(64, 3), torch.randn(64, 3)
    for mean in (False, True):
        loss, dz = simt.sse_loss(out, yy, 1.0 / 64 if mean else 1.0)
        rl, rdz = reference.loss_and_dz(out, yy, "mse" if mean else "sse", "none")
        torch.testing.assert_close(loss, rl, rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(dz, rdz, rtol=1e-5, atol=1e-6)
    logits, labels = torch.randn(200, 10) * 2, torch.randint(0, 10, (200,))
    loss, dl = simt.softmax_xent(logits, labels)
    rl, rdl = reference.softmax_xent(logits, labels)
    torch.testing.assert_close(loss, rl, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(dl, rdl, rtol=1e-4, atol=1e-6)
    # the one-block loss head on padded operands (what both GEMM-shaped trainers launch): gradient into a padded bf16 matrix,
    # head bias gradient, mean loss; rows / columns outside [rows, cols] untouched
    for rows, cols, ld in ((128, 10, 64), (1000, 2, 64), (5, 100, 128), (37, 128, 128)):
        big = torch.randn(rows + 3, ld) * 2
        lab = torch.randint(0, cols, (rows + 3,))
        dz = torch.full((rows + 3, ld), 7.0, dtype=torch.bfloat16)
        dlf = torch.full((rows + 3, ld), 7.0)
        db = torch.full((ld,), 7.0)
        loss = simt.softmax_xent_head(big, lab, rows, cols, dlf, dz, db)
        rl, rdl = reference.softmax_xent(big[:rows, :cols], lab[:rows])
        torch.testing.assert_close(loss, rl, rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(dlf[:rows, :cols], rdl, rtol=1e-4, atol=1e-6)
        assert torch.equal(dz[:rows, :cols], dlf[:rows, :cols].to(torch.bfloat16))
        torch.testing.assert_close(db[:cols], rdl.sum(0), rtol=1e-4, atol=1e-6)
        assert bool((dz[rows:] == 7).all()) and bool((dz[:, cols:] == 7).all()) and bool((db[cols:] == 7).all())
    prob = torch.rand(999).clamp(1e-4, 1 - 1e-4)
    tgt = (torch.rand(999) > 0.5).float()
    loss, correct = simt.eval_binary(prob, tgt)
    rl, rc = reference.eval_binary(prob.view(-1, 1), tgt.view(-1, 1))
    torch.testing.assert_close(loss, rl, rtol=1e-4, atol=1e-3)
    assert int(correct) == int(rc)
    x = torch.randn(300, 7)
    assert torch.equal(simt.argmax_rows(x), x.argmax(1, keepdim=True))
    feats = torch.rand(500, 10) * 7 - 2
    lo, hi = feats.min(0).values, feats.max(0).values
    torch.testing.assert_close(simt.minmax_scale(feats), (feats - lo) / (hi - lo), rtol=1e-5, atol=1e-6)


def test_feistel_permutation_transpose_and_ring_matmul_on_cpu(simt):
    perm = simt.feistel_permutation(1000, 3, 42)
    assert perm.shape == (3, 1000)
    for r in range(3):
        assert sorted(perm[r].tolist()) == list(range(1000))         # a bijection of [0, n) per row (cycle walking)
    assert not torch.equal(perm[0], perm[1]) and not torch.equal(perm[0], torch.arange(1000, dtype=torch.int32))
    assert torch.equal(perm, simt.feistel_permutation(1000, 3, 42)) and not torch.equal(perm, simt.feistel_permutation(1000, 3, 43))
    x = torch.randn(70, 45).to(torch.bfloat16)
    assert torch.equal(simt.transpose_bf16(x), x.t().contiguous())
    a = torch.randint(-2 ** 62, 2 ** 62, (9, 20))
    b = torch.randint(-2 ** 62, 2 ** 62, (20, 13))
    assert torch.equal(simt.ring_matmul(a, b), a @ b)                # arithmetic mod 2^64 (int64 wrap-around)


# ---- comm.cu on the CPU: W emulated ranks = W sets of buffers, kernels of different ranks run one after the other ----------
def test_star_round_kernel_on_cpu(simt):
    torch.manual_seed(1)
    W, P = 4, 1003                                            # P not a multiple of 4: scalar tail
    theta = torch.randn(P)
    weights = [0.4, 0.3, 0.2, 0.1]
    models = [torch.randn(P) for _ in range(W)]
    slots = torch.stack([w * m for w, m in zip(weights, models)])
    arrive = torch.full((W,), 5, dtype=torch.int32)
    inboxes, bflags = torch.zeros(W, P), torch.zeros(W, dtype=torch.int32)
    th = theta.clone()
    simt.star_round(th, slots, arrive, 5, inboxes, bflags, 6, 0b1111, 0.5, True, True, 3, 0.0, weights)
    want = theta + 0.5 * (sum(w * m for w, m in zip(weights, models)) - theta)
    torch.testing.assert_close(th, want, rtol=1e-5, atol=1e-5)
    assert all(torch.equal(inboxes[k], th) for k in range(W)) and bflags.tolist() == [6] * W
    # subset selection: only ranks 0 and 2 contribute / receive the broadcast
    inboxes.zero_(); bflags.zero_()
    th = theta.clone()
    sl = torch.stack([0.5 * models[0], torch.full((P,), 99.0), 0.5 * models[2], torch.full((P,), 99.0)])
    simt.star_round(th, sl, arrive, 5, inboxes, bflags, 6, 0b0101, 1.0, True, True, 2, 0.0, [0.5, 0, 0.5, 0])
    torch.testing.assert_close(th, 0.5 * (models[0] + models[2]), rtol=1e-5, atol=1e-5)
    assert torch.equal(inboxes[0], th) and torch.equal(inboxes[2], th) and float(inboxes[1].abs().max()) == 0 and bflags.tolist() == [6, 0, 6, 0]
    # deadline: rank 3 never arrives -> dropped after the timeout, the sum is renormalised over the weight that arrived
    late = torch.tensor([5, 5, 5, 4], dtype=torch.int32)
    th = theta.clone()
    mask = simt.star_round(th, slots, late, 5, inboxes, bflags, 7, 0b1111, 1.0, True, True, 3, 20.0, weights)
    assert mask == 0b0111
    torch.testing.assert_close(th, sum(w * m for w, m in zip(weights[:3], models[:3])) / 0.9, rtol=1e-4, atol=1e-5)
    # nobody arrives: theta is kept
    th = theta.clone()
    mask = simt.star_round(th, slots, torch.zeros(W, dtype=torch.int32), 5, inboxes, bflags, 8, 0b1111, 1.0, True, False, 2, 5.0, weights)
    assert mask == 0 and torch.equal(th, theta)


@pytest.mark.parametrize("server_lr", [1.0, 0.5])
def test_twoshot_fedavg_kernel_on_cpu(simt, server_lr):
    torch.manual_seed(2)
    W, n, chunk = 4, 4 * 350, 64                              # 22 chunks (the last one short), owner of chunk c = c % W
    weights = torch.tensor([0.1, 0.2, 0.3, 0.4])
    trained = torch.randn(W, n)
    prev = torch.randn(n)
    works = trained.clone()
    shadows = torch.zeros(W, n, dtype=torch.bfloat16)
    n_chunks = (n + chunk - 1) // chunk
    flags = torch.zeros(W, n_chunks, dtype=torch.int32)
    prevs = [prev.clone() for _ in range(W)]
    arrive = torch.full((W,), 3, dtype=torch.int32)
    for r in range(W):                                          # every rank reduces the chunks it owns and writes them everywhere
        simt.twoshot_fedavg(r, works, shadows, flags, arrive, weights, prevs[r] if server_lr != 1.0 else None, 3, 0b1111, server_lr, chunk, 2, None, 0.0)
    avg = (weights.view(-1, 1) * trained).sum(0)
    want = avg if server_lr == 1.0 else prev + server_lr * (avg - prev)
    for k in range(W):
        torch.testing.assert_close(works[k], want, rtol=1e-5, atol=1e-5)
        assert torch.equal(shadows[k], works[k].to(torch.bfloat16))
    assert int(flags.min()) == 3 and int(flags.max()) == 3


def test_twoshot_subset_and_reduce_push_on_cpu(simt):
    torch.manual_seed(3)
    W, n, chunk = 4, 512, 128
    trained = torch.randn(W, n)
    works = trained.clone()
    flags = torch.zeros(W, n // chunk, dtype=torch.int32)
    weights = torch.tensor([0.5, 0.0, 0.5, 0.0])
    arrive = torch.tensor([9, 0, 9, 0], dtype=torch.int32)      # ranks 1 and 3 are not selected and never arrive
    for r in range(W):
        simt.twoshot_fedavg(r, works, None, flags, arrive, weights, None, 9, 0b0101, 1.0, chunk, 1, None, 0.0)
    for k in range(W):                                          # every rank (selected or not) receives the new model
        torch.testing.assert_close(works[k], 0.5 * (trained[0] + trained[2]), rtol=1e-5, atol=1e-5)
    # many virtual clients per GPU: local sum of C pre-scaled client models pushed as one contribution
    C, P = 6, 1001
    slots, losses = torch.randn(C, P), torch.rand(C, 2)
    dst, loss_dst, flag = torch.zeros(P), torch.zeros(2), torch.zeros(1, dtype=torch.int32)
    simt.reduce_push(slots, dst, losses.reshape(-1).contiguous(), loss_dst, flag, 11, 3)
    torch.testing.assert_close(dst, slots.sum(0), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(loss_dst, losses.mean(0), rtol=1e-5, atol=1e-6)
    assert int(flag) == 11


# ---- convnet.cu on the CPU: the launchers and kernels themselves (grid-stride maps, two-phase blocks, the ticket-counter
# BatchNorm reduction with its atomics / fences), behind the same Python ops the GPU uses --------------------------------
def test_conv_kernels_on_cpu(simt):
    import test_conv_ops as T

    T.test_im2col_and_col2im_kernels("simt", (2, 64, 8, 8, 3, 1, 1))
    T.test_im2col_and_col2im_kernels("simt", (2, 64, 8, 8, 3, 2, 1))
    T.test_im2col_and_col2im_kernels("simt", (2, 16, 9, 7, 3, 2, 1))
    T.test_im2col_stem_reads_the_user_batch_directly("simt", "nchw_f32")
    T.test_pooling_kernels("simt", (2, 64, 16, 16, 3, 2, 1))
    T.test_pooling_kernels("simt", (1, 8, 6, 6, 2, 2, 0))
    T.test_pack_and_unpack_params("simt")
    T._splitk_reduce_case("simt", 16, 128, 640)
    T._splitk_reduce_case("simt", 5, 4, 12)


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("m,c,ldx", [(128, 64, 128), (2048, 128, 128), (100, 64, 64), (1030, 256, 256)])
def test_batchnorm_kernels_on_cpu(simt, m, c, ldx, fused):
    """``bn_reduce`` / ``bn_finalize`` / ``bn_apply`` / ``bn_bwd`` and (fused) ``bn_reduce_finalize_kernel`` — the single-launch
    reduction whose last block per channel group (atomic ticket, __threadfence) finalises and resets the counter."""
    import test_conv_ops as T

    T._batchnorm_case("simt", m, c, ldx, fused=fused)


# ---- gemm_wgmma.cu on the functional wgmma / TMA / mbarrier model (csrc/gemm_host_model.h) -------------------------------
def _gemm(simt, a, b, **kw):
    simt.gemm_tcgen05(a, b, kw.get("bias"), kw.get("relu", False), kw.get("relu_mask"), kw.get("out_bf16"), kw.get("out_f32"),
                      kw.get("out_bf16_t"), kw.get("sgd_master"), kw.get("sgd_lr", 0.0), kw.get("sgd_shadow"), kw.get("sgd_shadow_t"),
                      kw.get("colsum"), kw.get("tile_n", 0), kw.get("split_k", 0), kw.get("split_out"), kw.get("mn_m", 0),
                      kw.get("b_kn", False), kw.get("addend"), kw.get("conv", []), kw.get("produced", []))


def _bf(*shape):
    return torch.randn(*shape).to(torch.bfloat16)


def test_tcgen05_gemm_source_on_the_cpu_model_k_major(simt):
    """The persistent TMA -> wgmma -> staged epilogue pipeline (mbarrier phases, 4 "SMs" walking up to 8 tiles each) and
    every fused epilogue, against PyTorch."""
    torch.manual_seed(0)
    for m, n, k, tile_n in [(128, 128, 64, 0), (1024, 256, 192, 128), (512, 512, 128, 256), (256, 384, 64, 0)]:
        a, b = _bf(m, k), _bf(n, k)
        out = torch.full((m, n), 7.0)
        _gemm(simt, a, b, out_f32=out, tile_n=tile_n)
        torch.testing.assert_close(out, a.float() @ b.float().t(), rtol=1e-5, atol=1e-4)
    m, n, k = 256, 256, 128
    a, b, bias = _bf(m, k), _bf(n, k), torch.randn(n)
    acc = torch.relu(a.float() @ b.float().t() + bias)
    ob, ot, cs = torch.zeros(m, n, dtype=torch.bfloat16), torch.zeros(n, m, dtype=torch.bfloat16), torch.zeros(m // 32, n)
    _gemm(simt, a, b, bias=bias, relu=True, out_bf16=ob, out_bf16_t=ot, colsum=cs)
    assert torch.equal(ob, acc.to(torch.bfloat16)) and torch.equal(ot, ob.t().contiguous())
    torch.testing.assert_close(cs, acc.view(m // 32, 32, n).sum(1), rtol=1e-4, atol=1e-3)
    mask, add = _bf(m, n), _bf(m, n)
    of = torch.zeros(m, n)
    _gemm(simt, a, b, relu_mask=mask, addend=add, out_f32=of)
    torch.testing.assert_close(of, (a.float() @ b.float().t()) * (mask.float() > 0) + add.float(), rtol=1e-5, atol=1e-4)
    master0 = torch.randn(m, n)
    master, sh, sht = master0.clone(), torch.zeros(m, n, dtype=torch.bfloat16), torch.zeros(n, m, dtype=torch.bfloat16)
    _gemm(simt, a, b, sgd_master=master, sgd_lr=0.25, sgd_shadow=sh, sgd_shadow_t=sht)
    torch.testing.assert_close(master, master0 - 0.25 * (a.float() @ b.float().t()), rtol=1e-5, atol=1e-4)
    assert torch.equal(sh, master.to(torch.bfloat16)) and torch.equal(sht, sh.t().contiguous())
    # split-K: slices that do not divide the k-blocks evenly, more work units than CTAs
    a, b = _bf(256, 64 * 7), _bf(256, 64 * 7)
    part = torch.full((3 * 256 * 256 + 16,), 7.0)
    _gemm(simt, a, b, split_k=3, split_out=part)
    torch.testing.assert_close(part[: 3 * 256 * 256].view(3, 256, 256).sum(0), a.float() @ b.float().t(), rtol=1e-5, atol=1e-3)
    assert float(part[3 * 256 * 256:].min()) == 7.0
    want = torch.zeros(3 * 256 * 256)
    ops.gemm_bf16(a, b, split_k=3, split_out=want)                       # same slice boundaries as the CPU definition
    torch.testing.assert_close(part[: 3 * 256 * 256], want, rtol=1e-5, atol=1e-3)


def test_tcgen05_gemm_source_on_the_cpu_model_mn_major(simt):
    """MN-major wgmma operands (boxes of 64 rows x 64 columns, LBO 8192 / SBO 1024, +2048 bytes per wgmma): wgrad form AᵀB
    with TMA zero fill for the missing columns, dgrad form A·B[:K], with split-K and the fused SGD epilogue."""
    torch.manual_seed(1)
    for kd, ac, m, n in [(64, 128, 128, 128), (128, 64, 128, 128), (512, 64, 128, 640), (256, 256, 256, 256)]:
        a, b = _bf(kd, ac), _bf(kd, n)
        out = torch.full((m, n), 7.0)
        _gemm(simt, a, b, mn_m=m, out_f32=out)
        want = torch.zeros(m, n)
        want[:ac] = a.float().t() @ b.float()
        torch.testing.assert_close(out, want, rtol=1e-5, atol=1e-3)
    for m, kd, rows, n in [(128, 64, 64, 128), (256, 64, 128, 640), (128, 128, 128, 256)]:
        a, b = _bf(m, kd), _bf(rows, n)
        out = torch.zeros(m, n)
        _gemm(simt, a, b, b_kn=True, out_f32=out)
        torch.testing.assert_close(out, a.float() @ b[:kd].float(), rtol=1e-5, atol=1e-3)
    a, b = _bf(512, 64), _bf(512, 256)
    want = torch.zeros(128, 256)
    want[:64] = a.float().t() @ b.float()
    part = torch.zeros(4 * 128 * 256)
    _gemm(simt, a, b, mn_m=128, split_k=4, split_out=part)
    torch.testing.assert_close(part.view(4, 128, 256).sum(0), want, rtol=1e-5, atol=1e-3)
    master, sh = torch.ones(128, 256), torch.zeros(128, 256, dtype=torch.bfloat16)
    _gemm(simt, a, b, mn_m=128, sgd_master=master, sgd_lr=0.5, sgd_shadow=sh)
    torch.testing.assert_close(master, 1 - 0.5 * want, rtol=1e-5, atol=1e-3)
    assert torch.equal(sh, master.to(torch.bfloat16))


@pytest.mark.parametrize("n,h,w,cin,cout", [(4, 8, 8, 64, 64), (8, 4, 4, 128, 128), (32, 2, 2, 128, 64), (128, 1, 1, 64, 128), (8, 4, 4, 64, 128)])
def test_implicit_conv_kernels_on_the_cpu_model(simt, n, h, w, cin, cout):
    """Forward / dgrad (K-major W^T and packed MN-major weights, residual addend, 128x64 tile) / wgrad (MN-major 4-D boxes,
    fused SGD, split-K) of a stride-1 3x3 convolution: the producer's 4-D TMA boxes on the model against autograd."""
    from test_gpu_schedules import _implicit_case
    from colearn_federated_learning_b200.ops import conv as C

    d = _implicit_case(n, h, w, cin, cout)
    m, cp, kp = d["m"], d["cout_pad"], d["k_pad"]
    with C.simt():
        out = torch.full((m, cp), 7.0, dtype=torch.bfloat16)
        C.conv_gemm("fwd", d["act"], d["wp"], n, h, w, cin, 3, 3, 1, out_bf16=out)
        part = torch.zeros(3 * m * cp)
        C.conv_gemm("fwd", d["act"], d["wp"], n, h, w, cin, 3, 3, 1, split_k=3, split_out=part)
        add = torch.randn(m, cin).to(torch.bfloat16)
        dx, dx2 = torch.zeros(m, cin, dtype=torch.bfloat16), torch.zeros(m, cin, dtype=torch.bfloat16)
        C.conv_gemm("dgrad", d["dz"], d["wp"][:cout].t().contiguous(), n, h, w, cout, 3, 3, 1, out_bf16=dx, addend=add, rows_per_tap=cin)
        C.conv_gemm("dgrad", d["dz"], d["wp"], n, h, w, cout, 3, 3, 1, out_bf16=dx2, addend=add, rows_per_tap=cin, w_packed=True)
        master, sh = torch.zeros(cp, kp), torch.zeros(cp, kp, dtype=torch.bfloat16)
        C.conv_gemm("wgrad", d["act"], d["dz"], n, h, w, cin, 3, 3, 1, m_pad=cp, k_pad=kp, sgd_master=master, sgd_lr=-1.0, sgd_shadow=sh)
        s = max(2, min(4, m // 64))
        wpart = torch.zeros(s * cp * kp)
        C.conv_gemm("wgrad", d["act"], d["dz"], n, h, w, cin, 3, 3, 1, m_pad=cp, k_pad=kp, split_k=s, split_out=wpart)
    torch.testing.assert_close(out[:, :cout].float(), d["z"], rtol=2e-2, atol=3e-2)
    assert float(out[:, cout:].float().abs().max() if cp > cout else 0.0) == 0.0
    torch.testing.assert_close(part.view(3, m, cp).sum(0)[:, :cout], d["z"], rtol=1e-4, atol=1e-3)
    torch.testing.assert_close(dx.float(), d["dx"] + add.float(), rtol=2e-2, atol=5e-2)
    assert torch.equal(dx, dx2)                                              # same products, same accumulation order
    torch.testing.assert_close(master[:cout, :9 * cin], d["dw"], rtol=1e-4, atol=1e-3)
    assert float(master[cout:].abs().max() if cp > cout else 0.0) == 0.0 and float(master[:, 9 * cin:].abs().max() if kp > 9 * cin else 0.0) == 0.0
    assert torch.equal(sh, master.to(torch.bfloat16))
    torch.testing.assert_close(wpart.view(s, cp, kp).sum(0), master, rtol=1e-4, atol=1e-3)


@pytest.mark.skipif(__import__("os").environ.get("COLEARN_RUN_SLOW") != "1", reason="~4 minutes: set COLEARN_RUN_SLOW=1")
def test_whole_resnet18_step_from_kernel_sources_on_the_cpu_model(simt, monkeypatch):
    """One ResNet-18 SGD step (batch 128) with EVERY kernel — im2col / BatchNorm / pooling / packing, the wgmma GEMMs with
    their fused epilogues, the loss, the flat SGD — running from its CUDA source on the CPU (SIMT shim + wgmma / TMA model):
    (1) the default schedule agrees with the PyTorch definitions of the ops; (2) the schedule that has not run on a GPU
    yet (implicit GEMM level 2, MN-major wgrad, packed-weight dgrad, split-K, single-launch BatchNorm reduction) produces the
    same parameter update as the default schedule.  Measured on the authoring box: loss 2.58854 for both, update cosine
    1.000 between the schedules, 0.975 against the definitions (bf16 rounding points), 80-120 s per step."""
    from colearn_federated_learning_b200.fl.convnet import ConvNetTrainer
    from colearn_federated_learning_b200.models.resnet import ResNet18
    from colearn_federated_learning_b200.ops import conv as C

    torch.manual_seed(0)
    model = ResNet18(10)
    flat0 = flatten_params(model).clone()
    x, y = torch.randn(128, 3, 32, 32), torch.randint(0, 10, (128,))

    def run(on_model, **kw):
        flat = flat0.clone()
        tr = ConvNetTrainer(model, "cpu", 128, (32, 32), **kw)
        import contextlib
        with (C.simt() if on_model else contextlib.nullcontext()):
            tr.load(flat, None)
            loss = float(tr.step(x, y, 0.05))
            tr.store(flat, None)
        return (flat - flat0).double(), loss

    cos = lambda a, b: float((a * b).sum() / (a.norm() * b.norm()))  # noqa: E731
    d_def, l_def = run(False)
    d_src, l_src = run(True)
    assert abs(l_def - l_src) < 2e-2 and cos(d_def, d_src) > 0.95
    monkeypatch.setenv("COLEARN_CONV_FUSED_BN", "1")
    d_new, l_new = run(True, implicit=2, wgrad_mn=True, dgrad_kn=True, split_k=1)
    assert abs(l_new - l_src) < 1e-3 and cos(d_new, d_src) > 0.999


def test_racecheck_of_the_simt_kernels_on_cpu(tmp_path):
    """compute-sanitizer racecheck without a GPU (scripts/racecheck_cpu.sh): the persistent-MLP (every variant / net /
    batch mode), elementwise, comm and BatchNorm kernels are compiled for the CPU with -fsanitize=thread and run on small
    workloads — a shared-memory access pair that is not ordered by __syncthreads / a shuffle / a release-acquire flag would
    be reported as a data race.  (It found one: the weights-in-shared-memory variant's idle threads used to shadow-read
    the last neuron's row while its owner updated it; benign, fixed.)"""
    import os
    import shutil
    import subprocess

    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    probe = subprocess.run(["g++", "-fsanitize=thread", "-x", "c++", "-", "-o", str(tmp_path / "probe")], input="int main(){return 0;}",
                           capture_output=True, text=True)
    if probe.returncode != 0:
        pytest.skip("ThreadSanitizer runtime not available")
    p = subprocess.run(["sh", os.path.join(root, "scripts", "racecheck_cpu.sh"), str(tmp_path / "build")], capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, (p.stdout + p.stderr)[-4000:]
    assert "WARNING: ThreadSanitizer" not in p.stdout + p.stderr
    for part in ("mlp kernels ok", "elementwise kernels ok", "comm kernels ok", "conv kernels ok", "gemm kernels ok"):
        assert part in p.stdout


# ---- fused wgrad GEMM -> FedAvg reduce (csrc/produced.cuh): epilogue reports + produced_mark + twoshot_overlap_kernel ----------------
@pytest.mark.parametrize("chunk", [2048, 8192])
def test_fused_wgrad_to_twoshot_reduce_on_cpu(simt, chunk):
    """Two emulated ranks.  Each runs its last-step wgrad GEMM with the fused-SGD epilogue on a master matrix inside its
    arena; the epilogue warps report finished blocks, produced_mark covers the rest of the arena, and the overlapped
    two-shot (polling the produced tables instead of the arrive flags) then averages exactly the updated parameters."""
    from colearn_federated_learning_b200.ops.produced import ProducedSpec
    torch.manual_seed(11)
    W, M, N, K = 2, 256, 256, 128
    head, tail = 1000, 520                                      # arena = [head | master M x N | tail]; offsets not chunk-aligned
    n = head + M * N + tail
    assert n % 4 == 0
    n_chunks = (n + chunk - 1) // chunk
    works = torch.randn(W, n)
    start = works.clone()
    tables = torch.zeros(W, W, n_chunks, dtype=torch.int32)
    epoch = torch.tensor([6], dtype=torch.int32)                # published value = 6 + 1
    lr = 0.05
    want_rank = []
    for r in range(W):
        count = torch.zeros(n_chunks, dtype=torch.int32)
        flag_ptrs = [tables[o].data_ptr() for o in range(W)]
        sp = ProducedSpec.device(simt, count, flag_ptrs, epoch, 1, chunk_elems=chunk, n=n, rank=r, max_ctas=3)
        a, b = _bf(M, K), _bf(N, K)
        master = works[r, head:head + M * N].view(M, N)
        shadow = torch.zeros(M, N, dtype=torch.bfloat16)
        _gemm(simt, a, b, sgd_master=master, sgd_lr=lr, sgd_shadow=shadow, produced=sp.gemm_arg(head))
        w_want = start[r].clone()
        w_want[head:head + M * N] -= lr * (a.float() @ b.float().t()).reshape(-1)
        torch.testing.assert_close(works[r], w_want, rtol=1e-4, atol=1e-4)
        want_rank.append(w_want)
        # chunks fully inside the matrix are already published, the ones shared with head / tail are not
        inside = [c for c in range(n_chunks) if c * chunk >= head and min(n, (c + 1) * chunk) <= head + M * N]
        assert inside and all(int(tables[c % W, r, c]) == 7 for c in inside)
        edge = [c for c in range(n_chunks) if c not in inside]
        assert all(int(tables[c % W, r, c]) == 0 for c in edge)
        sp.mark(0, head)
        sp.mark(head + M * N, n)
        assert all(int(tables[c % W, r, c]) == 7 for c in range(n_chunks)) and sp.idle()
    # the overlapped two-shot: arrive flags are never raised, only the produced tables carry the epoch
    weights = torch.tensor([0.25, 0.75])
    flags = torch.zeros(W, n_chunks, dtype=torch.int32)
    arrive = torch.zeros(W, dtype=torch.int32)
    shadows = torch.zeros(W, n, dtype=torch.bfloat16)
    for r in range(W):
        simt.twoshot_fedavg(r, works, shadows, flags, arrive, weights, None, 7, 0b11, 1.0, chunk, 2, tables, 5.0)
    want = 0.25 * want_rank[0] + 0.75 * want_rank[1]
    for k in range(W):
        torch.testing.assert_close(works[k], want, rtol=1e-5, atol=1e-5)
        assert torch.equal(shadows[k], works[k].to(torch.bfloat16))
    assert int(flags.min()) == 7


def test_overlapped_twoshot_takes_chunks_as_they_are_produced(simt):
    """The overlapped kernel must not wait in chunk order: a producer thread publishes the chunks newest-first (the order
    of a backward pass) with pauses; the kernel finishes although chunk 0 only arrives last."""
    import threading
    import time
    torch.manual_seed(12)
    W, chunk, n = 2, 64, 64 * 9 + 20
    n_chunks = (n + chunk - 1) // chunk
    trained = torch.randn(W, n)
    works = trained.clone()
    tables = torch.zeros(W, W, n_chunks, dtype=torch.int32)
    tables[:, 1, :] = 4                                          # rank 1 is done with everything
    flags = torch.zeros(W, n_chunks, dtype=torch.int32)
    weights = torch.tensor([0.5, 0.5])
    arrive = torch.zeros(W, dtype=torch.int32)

    def producer():
        for c in range(n_chunks - 1, -1, -1):
            time.sleep(0.01)
            tables[c % W, 0, c] = 4

    th = threading.Thread(target=producer)
    th.start()
    simt.twoshot_fedavg(0, works, None, flags, arrive, weights, None, 4, 0b11, 1.0, chunk, 2, tables, 20.0)
    th.join()
    simt.twoshot_fedavg(1, works, None, flags, arrive, weights, None, 4, 0b11, 1.0, chunk, 2, tables, 20.0)
    for k in range(W):
        torch.testing.assert_close(works[k], trained.mean(0), rtol=1e-5, atol=1e-5)
    assert int(flags.min()) == 4




# ---- two-shot FedAvg with a deadline: arrived-set decision, ownership over the arrived ranks, second arena, resync ----------------
def test_twoshot_deadline_drops_a_late_rank_and_lets_it_resync(simt):
    """Kernel source on the CPU, three emulated ranks: rank 2 has not signalled when the coordinator's deadline expires.  The
    round completes on ranks 0 and 1 (weights renormalised, chunk ownership dealt between the two), every arena — the late
    rank's included — receives the result in its second arena, and the late rank, whose work arena was overwritten while it
    "trained", restores it from there before its next round."""
    W, n, chunk = 3, 4096 + 256, 1024
    n_chunks = (n + chunk - 1) // chunk
    torch.manual_seed(0)
    works = torch.randn(W, n)
    trained = works.clone()
    globals_ = torch.zeros(W, n)
    flags = torch.zeros(W, n_chunks, dtype=torch.int32)
    decisions = torch.zeros(W, 16, dtype=torch.int32)
    weights = torch.zeros(16)
    weights[:3] = torch.tensor([0.5, 0.3, 0.2])
    epoch = 5
    arrive = [torch.zeros(W, dtype=torch.int32) for _ in range(W)]
    for a in arrive:
        a[0] = a[1] = epoch                                   # ranks 0 and 1 finished their local fit; rank 2 did not
    def run_ranks(ranks, w, ep):                               # one emulated rank after the other, the coordinator (which decides) first
        for r in ranks:
            simt.twoshot_fedavg_deadline(r, w, globals_, flags, arrive[r], weights, ep, 0b111, chunk, 2, 2.0, decisions)

    run_ranks((0, 1), works, epoch)
    want = (0.5 * trained[0] + 0.3 * trained[1]) / 0.8        # renormalised over the arrived weight
    assert decisions[:, 2 * (epoch % 8)].tolist() == [epoch] * W and decisions[:, 2 * (epoch % 8) + 1].tolist() == [0b011] * W
    for k in range(W):
        torch.testing.assert_close(globals_[k], want, rtol=1e-6, atol=1e-6)
        torch.testing.assert_close(works[k], want, rtol=1e-6, atol=1e-6)
    assert bool((flags == epoch).all())
    # the late rank arrives afterwards: it is not in the decision, owns nothing, changes nothing
    works[2].normal_()                                        # (what its in-place training left behind)
    for a in arrive:
        a[2] = epoch
    before = (works[:2].clone(), globals_.clone())
    simt.twoshot_fedavg_deadline(2, works, globals_, flags, arrive[2], weights, epoch, 0b111, chunk, 2, 2.0, decisions)
    assert torch.equal(works[:2], before[0]) and torch.equal(globals_, before[1])
    # next round: rank 2 restores its arena from the second arena, the ranks that were in the decision do not
    w0 = works[0].clone()
    simt.twoshot_resync(decisions[2], epoch, 2, works[2], globals_[2])
    simt.twoshot_resync(decisions[0], epoch, 0, works[0], globals_[0].zero_())
    torch.testing.assert_close(works[2], want, rtol=1e-6, atol=1e-6)
    assert torch.equal(works[0], w0)
    # everybody in time: same result as the plain kernel, ownership over all three
    epoch += 1
    works2 = trained.clone()
    for a in arrive:
        a[:] = epoch
    run_ranks(range(W), works2, epoch)
    full = 0.5 * trained[0] + 0.3 * trained[1] + 0.2 * trained[2]
    for k in range(W):
        torch.testing.assert_close(works2[k], full, rtol=1e-6, atol=1e-6)
    assert decisions[:, 2 * (epoch % 8) + 1].tolist() == [0b111] * W
