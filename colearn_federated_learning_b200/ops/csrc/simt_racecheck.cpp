// Race check of the SIMT kernels on the CPU: the kernel sources (simt_mlp.cpp, simt_elementwise.cpp, simt_comm.cpp,
// simt_convnet.cpp = the .cu files through host_shim.h) are compiled with -fsanitize=thread and driven with small
// workloads.  Every CUDA thread is an OS thread, __syncthreads / shuffles are std::barrier synchronisation that
// ThreadSanitizer understands, shared memory is ordinary memory: a missing barrier between a shared-memory write and a
// read by another thread is reported as a data race — compute-sanitizer's racecheck, without a GPU.
// Built and run by scripts/racecheck_cpu.sh (tests/test_simt_emul.py::test_racecheck runs it when COLEARN_RUN_SLOW=1).
#define COLEARN_HOST_SHIM 1
#include <cstdio>
#include <cstdlib>
#include <chrono>
#include <thread>
#include <vector>

#include "colearn_kernels.h"

namespace {
float frand() { return (float)rand() / (float)RAND_MAX; }
std::vector<float> randv(size_t n, float scale = 1.f) {
  std::vector<float> v(n);
  for (auto& x : v) x = (frand() - 0.5f) * 2.f * scale;
  return v;
}
#define CK(e)                                                   \
  do {                                                          \
    if ((e) != cudaSuccess) {                                   \
      fprintf(stderr, "launch failed: %s\n", #e);               \
      return 1;                                                 \
    }                                                           \
  } while (0)
}  // namespace

int main() {
  using namespace colearn;
  srand(1);
  // ---- persistent MLP: every net x variant, batch 1 and batch 3 (gradient-accumulation path), two clients ----------------
  const int din[5] = {10, 10, 2, 10, 10}, dout[5] = {1, 2, 1, 10, 5};
  const int losses[5] = {LOSS_BCE, LOSS_XENT, LOSS_SSE, LOSS_MSE, LOSS_XENT};
  for (int kind = 0; kind < 5; ++kind)
    for (int variant : {1, 3, 5, 6})
      for (int batch : {1, 3}) {
        const int P = mlp_net_num_params(kind), n = 7;
        std::vector<float> theta = randv(P, 0.3f), x = randv((size_t)n * din[kind]), y((size_t)n * (losses[kind] == LOSS_XENT ? 1 : dout[kind]));
        for (auto& v : y) v = (float)(rand() % 2);
        std::vector<float> out0(P), out1(P), loss(4);
        std::vector<ClientDesc> d(2);
        for (int c = 0; c < 2; ++c) {
          memset(&d[c], 0, sizeof(ClientDesc));
          d[c].x = x.data(); d[c].y = y.data(); d[c].theta_in = theta.data();
          d[c].theta_out = c ? out1.data() : out0.data(); d[c].loss_out = loss.data() + 2 * c;
          d[c].n = n; d[c].perm_rows = 1; d[c].y_dim = losses[kind] == LOSS_XENT ? 1 : dout[kind]; d[c].out_scale = 0.5f;
        }
        SgdHyper hp{batch, 2, -1, losses[kind], 0.05f, variant};
        CK(launch_mlp_local_sgd(kind, d.data(), 2, hp, nullptr));
        std::vector<float> o((size_t)n * dout[kind]);
        CK(launch_mlp_forward(kind, theta.data(), x.data(), o.data(), n, nullptr));
      }
  printf("mlp kernels ok\n");
  // ---- elementwise (the ones with shared memory / shuffles / atomics) ----------------------------------------------------------
  {
    const int64_t n = 3000;
    std::vector<float> z = randv(n), yv(n), dz(n), loss(1);
    for (auto& v : yv) v = (float)(rand() % 2);
    CK(launch_sigmoid_bce(z.data(), yv.data(), dz.data(), loss.data(), n, nullptr));
    CK(launch_sse(z.data(), yv.data(), dz.data(), loss.data(), n, 1.f, nullptr));
    std::vector<float> logits = randv(100 * 10), dl(1000);
    std::vector<int64_t> labels(100);
    for (auto& l : labels) l = rand() % 10;
    CK(launch_softmax_xent(logits.data(), 0, labels.data(), dl.data(), nullptr, loss.data(), 100, 10, nullptr));
    std::vector<float> hb(10);
    std::vector<__nv_bfloat16> dl16(1000);
    CK(launch_softmax_xent_head(logits.data(), 0, 10, labels.data(), dl.data(), 10, dl16.data(), 10, hb.data(), loss.data(), 100, 10, nullptr));
    std::vector<float> p(n);
    for (auto& v : p) v = 0.01f + 0.98f * frand();
    int correct = 0;
    CK(launch_eval_binary(p.data(), yv.data(), loss.data(), &correct, n, nullptr));
    std::vector<int64_t> am(100);
    CK(launch_argmax_rows(logits.data(), am.data(), 100, 10, nullptr));
    // detection-metrics summary: matched shared-memory counts, segment switches inside a CTA (flush), the ticket finalisation;
    // C = 1 over 3 uneven segments (one empty) on 2 CTAs, then C = 10
    {
      const int64_t offs[4] = {0, 2100, 2100, 3000};
      std::vector<int64_t> table;
      const int64_t units = es_build_table(offs, 3, table);
      std::vector<float> ylab(3000);
      for (auto& v : ylab) v = (float)(rand() % 10);
      std::vector<int64_t> out1(es_out_words(3, 1, 64, units)), out10(es_out_words(3, 10, 64, units));
      EvalSummaryArgs ea{p.data(), yv.data(), table.data(), 3, units, 1, 64, 0.5f, out1.data()};
      CK(launch_eval_summary(ea, 2, nullptr));
      std::vector<float> z10 = randv(3000 * 10);
      EvalSummaryArgs eb{z10.data(), ylab.data(), table.data(), 3, units, 10, 64, 0.5f, out10.data()};
      CK(launch_eval_summary(eb, 2, nullptr));
      // reconstruction-error summary: the same segments on 2 CTAs, labels and per-row outputs
      std::vector<float> xh = randv(3000 * 10), xr = randv(3000 * 10), err(3000);
      std::vector<uint8_t> flag(3000);
      std::vector<int64_t> outr(rs_out_words(3, 64, units));
      ReconSummaryArgs ra{xh.data(), xr.data(), yv.data(), table.data(), 3, units, 10, 64, 40, err.data(), flag.data(), outr.data()};
      CK(launch_recon_summary(ra, 2, nullptr));
    }
    std::vector<float> feats = randv(200 * 10), scaled(2000);
    CK(launch_minmax_scale(feats.data(), scaled.data(), 200, 10, nullptr));
    std::vector<__nv_bfloat16> tin(70 * 45), tout(70 * 45);
    for (auto& v : tin) v = __float2bfloat16(frand());
    CK(launch_transpose_bf16(tin.data(), tout.data(), 70, 45, nullptr));
    std::vector<long long> A(9 * 20, 3), B(20 * 13, 5), C(9 * 13);
    CK(launch_ring_matmul(A.data(), B.data(), C.data(), 9, 20, 13, nullptr));
    // uplink codec: encode 3 rows (warp max by shuffles), then the fused decode + FedAvg (weights in shared memory) and its
    // robust twin, int8 and int4, with a partial last block
    const int64_t qn = 1000, qrow = 1008;
    std::vector<float> qtheta = randv(qn), qmodels = randv(3 * qn), qscales(3 * 4), qw(3, 1.f / 3);
    std::vector<uint32_t> qkeys = {1u, 2u, 3u};
    alignas(16) static uint8_t qpayload[3 * 1008];
    // every fused apply below: the plain step (sgd, lr 1), the mean unless it says otherwise, no work buffer unless it needs one
    ServerOptArgs sgd;
    memset(&sgd, 0, sizeof(sgd));
    sgd.lr = 1.f;
    const AggregatorArgs mean{AGG_MEAN, 0.f, 0, 0.f, 0.f}, median{AGG_MEDIAN, 0.f, 0, 0.f, 0.f};
    const ApplyWork nowork{nullptr, nullptr, 0};
    for (int bits : {8, 4}) {
      CK(launch_quantize_delta(qmodels.data(), qn, qtheta.data(), qkeys.data(), 3, bits, qpayload, qrow, qscales.data(), qn, nullptr));
      ClientRows q{};
      q.format = bits == 8 ? ROWS_INT8 : ROWS_INT4; q.k = 3; q.stride = qrow; q.weights = qw.data(); q.payload = qpayload; q.scales = qscales.data();
      CK(launch_fedavg_apply(qtheta.data(), q, mean, sgd, qn, nowork, nullptr));
      CK(launch_fedavg_apply(qtheta.data(), q, median, sgd, qn, nowork, nullptr));
    }
    // top-k uplink: encode 3 rows (warp select by reductions and ballots, residual written back), then the sparse decode +
    // FedAvg (per-warp shared accumulator, one __syncwarp per slot), k = 8, with a partial last block (m_last = 232)
    std::vector<float> kres(3 * qn, 0.f), kvals(3 * 32);
    std::vector<uint8_t> kidx(3 * 32);
    CK(launch_topk_delta(qmodels.data(), qn, qtheta.data(), kres.data(), qn, 3, 8, kidx.data(), kvals.data(), 32, qn, nullptr));
    ClientRows kr{};
    kr.format = ROWS_TOPK; kr.k = 3; kr.stride = 32; kr.weights = qw.data(); kr.indices = kidx.data(); kr.values = kvals.data(); kr.topk = 8;
    CK(launch_fedavg_apply(qtheta.data(), kr, mean, sgd, qn, nowork, nullptr));
    // compressed downlink: encode-and-advance of one replica (block max by shuffles / warp select, replica written in place),
    // then the device-side apply of the same wire to a second replica, int8, int4 and topk k = 8, partial last block
    std::vector<float> drep(qn, 0.f), dev_rep(qn, 0.f);
    for (int bits : {8, 4}) {
      CK(launch_downlink_quant(qtheta.data(), drep.data(), 7u, bits, qpayload, qrow, qscales.data(), qn, nullptr));
      CK(launch_replica_apply_quant(dev_rep.data(), qpayload, qrow, qscales.data(), bits, qn, nullptr));
    }
    CK(launch_downlink_topk(qtheta.data(), drep.data(), 8, kidx.data(), kvals.data(), qn, nullptr));
    CK(launch_replica_apply_topk(dev_rep.data(), kidx.data(), kvals.data(), 8, qn, nullptr));
    // secure aggregation: the mask of one row (counts by warp reductions and atomics, partial last column), then the unmask-apply
    // on the fused path (few streams) and on the split path (many streams: atomicAdd into the scratch row, then the finalize)
    alignas(16) static uint32_t skeys[40 * 8];
    std::vector<int> ssigns(40), scounts(2);
    for (int i = 0; i < 40 * 8; ++i) skeys[i] = (uint32_t)rand() * 2654435761u;
    for (int i = 0; i < 40; ++i) ssigns[i] = (i & 1) ? -1 : 1;
    std::vector<uint32_t> smasked(2 * qn);
    alignas(16) static uint32_t swork[1000];
    CK(launch_secagg_mask(qmodels.data(), qtheta.data(), skeys, ssigns.data(), 3, 0.5f, 20, smasked.data(), scounts.data(), qn, nullptr));
    CK(launch_secagg_mask(qmodels.data() + qn, qtheta.data(), skeys, ssigns.data(), 3, 0.5f, 20, smasked.data() + qn, scounts.data(), qn,
                          nullptr));
    ClientRows sr{};
    sr.format = ROWS_SECAGG; sr.k = 2; sr.stride = qn; sr.masked = smasked.data(); sr.keys = skeys; sr.signs = ssigns.data();
    sr.frac_bits = 20; sr.n_mean = 2;
    for (int streams : {4, 40}) {
      sr.streams = streams;
      CK(launch_fedavg_apply(qtheta.data(), sr, mean, sgd, qn, ApplyWork{swork, nullptr, 0}, nullptr));
    }
    // distance-based aggregation: geomed L = 3 (distance pass, ticket finalisation by the last CTA, two fused centre passes on the
    // register path and the general one, apply) and norm_clip, fp32 and int8 rows, partial last chunk
    {
      const int64_t dn = 2100;
      std::vector<float> dtheta = randv(dn), drows = randv(40 * dn), dalpha(40, 1.f / 40), dw(40);
      const AggregatorArgs geo{DAGG_GEOMED, 0.f, 3, 1e-6f, 0.f}, clip{DAGG_NORM_CLIP, 0.f, 1, 0.f, 0.5f};
      ClientRows fr{}, qr{};
      fr.format = ROWS_F32; fr.k = 40; fr.stride = dn; fr.weights = dalpha.data(); fr.models = drows.data();
      qr.format = ROWS_INT8; qr.k = 3; qr.stride = qrow; qr.weights = dalpha.data(); qr.payload = qpayload; qr.scales = qscales.data();
      std::vector<double> dscratch(fedavg_apply_work_bytes(fr, geo, dn) / 8 + 2);
      const ApplyWork dwork{dscratch.data(), dw.data(), 2};
      for (int dk : {5, 40}) {
        fr.k = dk;
        CK(launch_fedavg_apply(dtheta.data(), fr, geo, sgd, dn, dwork, nullptr));
        CK(launch_fedavg_apply(dtheta.data(), fr, clip, sgd, dn, dwork, nullptr));
        CK(launch_fedavg_apply(dtheta.data(), qr, geo, sgd, qn, dwork, nullptr));
      }
      // asynchronous buffered aggregation: fp32 rows read as deltas to ring slots, the new theta stored to the write slot by the
      // mean (weights in shared memory), the robust body and the distance passes
      alignas(16) static float ring[3 * 2100];
      std::vector<int> bases = {0, 2, 0, 2, 0};
      ClientRows br{};
      br.format = ROWS_F32_BASED; br.k = 5; br.stride = dn; br.weights = dalpha.data(); br.models = drows.data();
      br.ring = ring; br.ring_slots = 3; br.write_slot = 1; br.base_slot = br.base_slot_host = bases.data();
      CK(launch_fedavg_apply(dtheta.data(), br, mean, sgd, dn, nowork, nullptr));
      CK(launch_fedavg_apply(dtheta.data(), br, median, sgd, dn, nowork, nullptr));
      CK(launch_fedavg_apply(dtheta.data(), br, geo, sgd, dn, dwork, nullptr));
    }
  }
  printf("elementwise kernels ok\n");
  // ---- comm: star round (with deadline) and two-shot on 3 emulated ranks, reduce_push -------------------------------------------
  {
    const int W = 3, P = 1003;
    std::vector<float> theta = randv(P), slots = randv((size_t)W * P), inbox((size_t)W * P);
    std::vector<uint32_t> arrive(W, 5), bflags(W, 0), decision(2, 0);
    uint32_t counter = 0;
    StarRoundArgs a;
    memset(&a, 0, sizeof(a));
    a.theta = theta.data(); a.slots = slots.data(); a.slot_stride = P; a.arrive_flags = arrive.data(); a.arrive_epoch = 5;
    for (int k = 0; k < W; ++k) { a.peer_inbox[k] = inbox.data() + (size_t)k * P; a.peer_bcast_flag[k] = &bflags[k]; a.weights[k] = 1.f / W; }
    a.bcast_epoch = 6; a.select_mask = 7; a.world = W; a.server_lr = 1.f; a.n = P; a.do_reduce = 1; a.do_bcast = 1;
    a.grid_counter = &counter; a.timeout_ns = 5000000ull; a.decision = decision.data();
    CK(launch_star_round(a, 3, nullptr));
    // the same round with a server optimizer (FedAdam): moments read and written next to theta, float4 body + scalar tail
    std::vector<float> m(P, 0.f), v(P, 1e-6f);
    a.opt.kind = SOPT_ADAM; a.opt.lr = 0.01f; a.opt.beta1 = 0.9f; a.opt.beta2 = 0.99f; a.opt.tau = 1e-3f;
    a.opt.m = m.data(); a.opt.v = v.data(); a.arrive_epoch = 5; a.bcast_epoch = 7;
    CK(launch_star_round(a, 3, nullptr));
    // the same round with a robust aggregator (median of the raw slots, register rank count), float4 body + scalar tail
    memset(&a.opt, 0, sizeof(a.opt));
    a.agg.kind = AGG_MEDIAN; a.bcast_epoch = 8;
    CK(launch_star_round(a, 3, nullptr));
    memset(&a.agg, 0, sizeof(a.agg));
    const int64_t n = 4 * 200, chunk = 64;
    std::vector<float> works = randv((size_t)W * n), weights(W, 1.f / W);
    std::vector<uint32_t> cflags((size_t)W * ((n + chunk - 1) / chunk), 0), arr(W, 2);
    for (int r = 0; r < W; ++r) {
      TwoShotArgs t;
      memset(&t, 0, sizeof(t));
      for (int k = 0; k < W; ++k) { t.work[k] = works.data() + (size_t)k * n; t.chunk_flags[k] = cflags.data() + (size_t)k * ((n + chunk - 1) / chunk); }
      t.arrive_flags = arr.data(); t.weights = weights.data(); t.epoch = 2; t.select_mask = 7; t.server_lr = 1.f; t.n = n; t.chunk_elems = chunk;
      t.world = W; t.rank = r;
      CK(launch_twoshot_fedavg(t, 2, nullptr));
    }
    // two-shot with FedAdam: every rank keeps theta_prev and the moments of the chunks it owns
    std::vector<float> prevs = randv((size_t)W * n), ms((size_t)W * n, 0.f), vs((size_t)W * n, 1e-6f);
    for (int r = 0; r < W; ++r) {
      TwoShotArgs t;
      memset(&t, 0, sizeof(t));
      for (int k = 0; k < W; ++k) { t.work[k] = works.data() + (size_t)k * n; t.chunk_flags[k] = cflags.data() + (size_t)k * ((n + chunk - 1) / chunk); }
      t.arrive_flags = arr.data(); t.weights = weights.data(); t.epoch = 2; t.select_mask = 7; t.server_lr = 0.01f; t.n = n; t.chunk_elems = chunk;
      t.world = W; t.rank = r; t.theta_prev = prevs.data() + (size_t)r * n;
      t.opt.kind = SOPT_ADAM; t.opt.lr = 0.01f; t.opt.beta1 = 0.9f; t.opt.beta2 = 0.99f; t.opt.tau = 1e-3f;
      t.opt.m = ms.data() + (size_t)r * n; t.opt.v = vs.data() + (size_t)r * n;
      CK(launch_twoshot_fedavg(t, 2, nullptr));
    }
    // two-shot with a trimmed mean: the owner ranks its peers' values in registers (P2P path)
    for (int r = 0; r < W; ++r) {
      TwoShotArgs t;
      memset(&t, 0, sizeof(t));
      for (int k = 0; k < W; ++k) { t.work[k] = works.data() + (size_t)k * n; t.chunk_flags[k] = cflags.data() + (size_t)k * ((n + chunk - 1) / chunk); }
      t.arrive_flags = arr.data(); t.weights = weights.data(); t.epoch = 2; t.select_mask = 7; t.server_lr = 1.f; t.n = n; t.chunk_elems = chunk;
      t.world = W; t.rank = r;
      t.agg.kind = AGG_TRIMMED_MEAN; t.agg.trim = 0.34f;
      CK(launch_twoshot_fedavg(t, 2, nullptr));
    }
    std::vector<float> dst(P), lsrc = randv(2 * W), ldst(2);
    uint32_t flag = 0, cnt2 = 0;
    CK(launch_reduce_push(slots.data(), W, P, P, dst.data(), lsrc.data(), ldst.data(), &flag, 9, &cnt2, 3, nullptr));
  }
  printf("comm kernels ok\n");
  // ---- convnet: the two-phase BatchNorm reductions (shared memory + ticket counter) ------------------------------------------------
  {
    using namespace convops;
    const int M = 300, C = 128;
    std::vector<__nv_bfloat16> x((size_t)M * C), dy((size_t)M * C), out((size_t)M * C);
    for (size_t i = 0; i < x.size(); ++i) { x[i] = __float2bfloat16(frand()); dy[i] = __float2bfloat16(frand() - 0.5f); out[i] = __float2bfloat16(frand() - 0.3f); }
    std::vector<float> partial(2 * C * 64), mean(C), invstd(C), rm(C), rv(C, 1.f);
    std::vector<unsigned> counters(C / 64, 0);
    BnReduceArgs r;
    memset(&r, 0, sizeof(r));
    r.mode = 0; r.x = x.data(); r.ldx = C; r.M = M; r.C = C; r.rows_per_block = 32; r.partial = partial.data();
    BnFinalizeArgs f;
    memset(&f, 0, sizeof(f));
    f.mode = 0; f.partial = partial.data(); f.nseg = bn_nseg(r); f.M = M; f.C = C; f.eps = 1e-5f; f.momentum = 0.1f;
    f.mean = mean.data(); f.invstd = invstd.data(); f.running_mean = rm.data(); f.running_var = rv.data();
    CK(launch_bn_reduce(r, nullptr));
    CK(launch_bn_finalize(f, nullptr));
    BnFusedArgs fa{r, f, counters.data()};
    CK(launch_bn_reduce_finalize(fa, nullptr));
    r.mode = 1; r.dy = dy.data(); r.out = out.data(); r.mean = mean.data(); r.invstd = invstd.data();
    std::vector<float> dg(C), db(C);
    f.mode = 1; f.dgamma = dg.data(); f.dbeta = db.data();
    BnFusedArgs fb{r, f, counters.data()};
    CK(launch_bn_reduce_finalize(fb, nullptr));
  }
  printf("conv kernels ok\n");
  // ---- wgmma GEMM on the functional model: the TMA -> MMA -> epilogue pipeline is ordered by mbarriers only -------------------
  {
    auto bf = [](size_t n) { std::vector<__nv_bfloat16> v(n); for (auto& x : v) x = __float2bfloat16(frand() - 0.5f); return v; };
    GemmEpilogue ep;
    // K-major: 16 tiles on 4 CTAs (both accumulator stages, smem ring wrap-around), then split-K
    {
      const int M = 512, N = 512, K = 64 * 5;
      auto a = bf((size_t)M * K), b = bf((size_t)N * K);
      std::vector<float> out((size_t)M * N), part((size_t)3 * M * N);
      memset(&ep, 0, sizeof(ep)); ep.ready_chunk_elems = 1; ep.out_f32 = out.data(); ep.tile_n = 128;
      CK(launch_gemm_tcgen05(a.data(), b.data(), M, N, K, ep, nullptr));
      memset(&ep, 0, sizeof(ep)); ep.ready_chunk_elems = 1; ep.split_k = 3; ep.split_out = part.data();
      CK(launch_gemm_tcgen05(a.data(), b.data(), M, N, K, ep, nullptr));
    }
    // MN-major wgrad form with the fused SGD epilogue
    {
      const int Kd = 256, ac = 64, M = 128, N = 384;
      auto a = bf((size_t)Kd * ac), b = bf((size_t)Kd * N);
      std::vector<float> master((size_t)M * N, 1.f);
      std::vector<__nv_bfloat16> shadow((size_t)M * N);
      memset(&ep, 0, sizeof(ep)); ep.ready_chunk_elems = 1; ep.sgd_master = master.data(); ep.sgd_lr = 0.1f; ep.sgd_shadow = shadow.data();
      CK(launch_gemm_tcgen05_mn(a.data(), 1, ac, b.data(), Kd, M, N, Kd, ep, nullptr));
    }
    // implicit-GEMM forward: 4 images of 8x8, 64 -> 64 channels
    {
      const int n = 4, H = 8, W = 8, C = 64, M = n * H * W, N = 128, K = 9 * C;
      auto act = bf((size_t)M * C), wp = bf((size_t)N * 640);
      std::vector<__nv_bfloat16> out((size_t)M * N);
      memset(&ep, 0, sizeof(ep)); ep.ready_chunk_elems = 1; ep.out_bf16 = out.data();
      ep.conv.mode = 1; ep.conv.C = C; ep.conv.KH = 3; ep.conv.KW = 3; ep.conv.pad = 1; ep.conv.HW = H * W; ep.conv.n_images = n;
      CK(launch_gemm_tcgen05_conv(act.data(), n, H, W, wp.data(), N, 640, M, N, K, ep, nullptr));
    }
    // epilogue modes with transposed copies (dgrad: mask + transposed output + column sums; wgrad: fused SGD + both shadows)
    {
      const int M = 256, N = 256, K = 128;
      auto a = bf((size_t)M * K), b = bf((size_t)N * K), mask = bf((size_t)M * N);
      std::vector<__nv_bfloat16> out((size_t)M * N), out_t((size_t)M * N);
      std::vector<float> cs((size_t)(M / 32) * N), master((size_t)M * N, 1.f);
      memset(&ep, 0, sizeof(ep)); ep.ready_chunk_elems = 1; ep.relu_mask = mask.data(); ep.out_bf16 = out.data();
      ep.out_bf16_t = out_t.data(); ep.colsum = cs.data();
      CK(launch_gemm_tcgen05(a.data(), b.data(), M, N, K, ep, nullptr));
      memset(&ep, 0, sizeof(ep)); ep.ready_chunk_elems = 1; ep.sgd_master = master.data(); ep.sgd_lr = 0.1f;
      ep.sgd_shadow = out.data(); ep.sgd_shadow_t = out_t.data(); ep.tile_n = 256;
      CK(launch_gemm_tcgen05(a.data(), b.data(), M, N, K, ep, nullptr));
    }
    // fused wgrad -> FedAvg reduce: fused-SGD epilogue with per-chunk reports into an unaligned arena, marks for the rest, then the
    // overlapped two-shot of two ranks while a host thread publishes rank 1's chunks newest-first
    {
      const int W = 2, M = 256, N = 256, Kd = 128, head = 1000, tail = 520, shift = 11;
      const int64_t n = head + (int64_t)M * N + tail, chunk = 1 << shift, n_chunks = (n + chunk - 1) / chunk;
      std::vector<float> works((size_t)W * n, 0.5f), weights(W, 0.5f);
      std::vector<uint32_t> tables((size_t)W * W * n_chunks, 0), count(n_chunks, 0), cflags((size_t)W * n_chunks, 0), arr(W, 0), epoch(1, 8);
      auto a = bf((size_t)M * Kd), b = bf((size_t)N * Kd);
      ProducedSignal sig;
      memset(&sig, 0, sizeof(sig));
      sig.count = count.data(); sig.epoch_ptr = epoch.data(); sig.epoch_add = 1; sig.n = n; sig.chunk_shift = shift; sig.world = W; sig.rank = 0; sig.n_chunks = (int)n_chunks;
      for (int o = 0; o < W; ++o) sig.flags[o] = tables.data() + (size_t)o * W * n_chunks;
      memset(&ep, 0, sizeof(ep)); ep.ready_chunk_elems = 1; ep.sgd_master = works.data() + head; ep.sgd_lr = 0.1f;
      ep.produced = &sig; ep.produced_elem_offset = head; ep.max_ctas = 3;
      CK(launch_gemm_tcgen05(a.data(), b.data(), M, N, Kd, ep, nullptr));
      CK(launch_produced_mark(&sig, shift, 0, head, nullptr));
      CK(launch_produced_mark(&sig, shift, head + (int64_t)M * N, n, nullptr));
      for (int64_t c = 0; c < n_chunks; ++c)
        if (tables[(size_t)(c % W) * W * n_chunks + c] != 9 || count[c] != 0) { fprintf(stderr, "chunk %lld not published\n", (long long)c); return 1; }
      std::thread producer([&] {
        for (int64_t c = n_chunks - 1; c >= 0; --c) {
          std::this_thread::sleep_for(std::chrono::milliseconds(2));
          __atomic_store_n(&tables[(size_t)(c % W) * W * n_chunks + (size_t)1 * n_chunks + c], 9u, __ATOMIC_RELEASE);
        }
      });
      for (int r = 0; r < W; ++r) {
        TwoShotArgs t;
        memset(&t, 0, sizeof(t));
        for (int k = 0; k < W; ++k) { t.work[k] = works.data() + (size_t)k * n; t.chunk_flags[k] = cflags.data() + (size_t)k * n_chunks; }
        t.arrive_flags = arr.data(); t.weights = weights.data(); t.epoch = 9; t.select_mask = 3; t.server_lr = 1.f; t.n = n; t.chunk_elems = chunk;
        t.world = W; t.rank = r; t.produced = tables.data() + (size_t)r * W * n_chunks; t.produced_timeout_ns = 20000000000ull;
        CK(launch_twoshot_fedavg(t, 2, nullptr));
      }
      producer.join();
    }
  }
  printf("gemm kernels ok\n");
  return 0;
}
