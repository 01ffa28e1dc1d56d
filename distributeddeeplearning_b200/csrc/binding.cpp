// pybind11 bindings of the b200-ddl native runtime and kernels.
//
// Deliberately torch-header-free: tensors cross the boundary as raw device pointers
// (tensor.data_ptr()) and a stream handle (torch.cuda.current_stream().cuda_stream); shape /
// dtype / contiguity checks live in the Python wrappers (ops/*.py, parallel/engine.py).  This keeps
// the build to seconds and the module importable on a GPU-less box.
#include <pybind11/pybind11.h>
#include <pybind11/functional.h>
#include <pybind11/stl.h>

#include <cuda_runtime.h>

#include <stdexcept>
#include <string>
#include <tuple>
#include <vector>

#include "comm/comm.h"
#include "ops/conv_gemm.cuh"
#include "ops/ops.h"
#include "runtime/host_runtime.h"
#include "runtime/step_launcher.h"

namespace py = pybind11;
using ddl::BnBwdArgs;
using ddl::BnFwdArgs;
using ddl::BucketArgs;
using ddl::CommCtx;
using ddl::ConvArgs;
using ddl::PoolArgs;
using ddl::SgdHyper;
using ddl::WgradArgs;
using ddl::XentArgs;

namespace ddl {
cudaError_t launch_conv_gemm(int mode, const ConvArgs& a, const void* w, int w_rows, int w_cols, int n_total,
                             const void* a_matrix, int a_cols, cudaStream_t stream);
cudaError_t launch_conv_wgrad(const WgradArgs& a, const void* dy, const void* x_matrix, int splits,
                              cudaStream_t stream);
cudaError_t launch_expand_grouped_weight(const void* w, void* out, int cout, int taps, int gw, cudaStream_t stream);
void set_conv_force_stages(int s);
void set_wgrad_swap(int on);
void set_conv_persistent(int on);
void set_conv_cluster(int on);
void set_conv_deep(int on);
void set_pdl(int on);
void set_bn_reverse(int on);
void set_conv_wait_hint(int ns);
cudaError_t conv_timeout_info(unsigned int out[8]);
}  // namespace ddl

namespace {

using ptr_t = uintptr_t;

template <class T>
T* P(ptr_t p) { return reinterpret_cast<T*>(p); }
cudaStream_t S(ptr_t s) { return reinterpret_cast<cudaStream_t>(s); }

void check(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}

struct PyCommCtx {
  CommCtx c{};
};

PoolArgs pool_args(int N, int H, int W, int C, int Pq, int Q, int k, int stride, int pad) {
  PoolArgs p;
  p.N = N; p.H = H; p.W = W; p.C = C; p.P = Pq; p.Q = Q; p.k = k; p.stride = stride; p.pad = pad;
  return p;
}

}  // namespace

PYBIND11_MODULE(_C, m) {
  m.doc() = "ddl native runtime + sm_90a kernels";
  m.attr("MAX_COMM_BLOCKS") = ddl::kMaxCommBlocks;
  m.attr("COMM_CHANNELS") = ddl::kCommChannels;
  m.attr("SIGNAL_PAD_BYTES") = ddl::kSignalPadBytes;
  m.attr("SGD_HYPER_BYTES") = sizeof(SgdHyper);
  m.attr("CONV_FWD") = static_cast<int>(ddl::kConvFwd);
  m.attr("CONV_DGRAD") = static_cast<int>(ddl::kConvDgrad);
  m.attr("CONV_GEMM") = static_cast<int>(ddl::kConvGemm);
  m.attr("CONV_STEM") = static_cast<int>(ddl::kConvStem);
  m.attr("CONV_TILE_FWD") = static_cast<int>(ddl::kConvTileFwd);
  m.attr("CONV_STEM_TMA") = static_cast<int>(ddl::kConvStemTma);
  m.attr("CONV_TILE_DGRAD") = static_cast<int>(ddl::kConvTileDgrad);
  m.attr("CONV_GEMM_DGRAD") = static_cast<int>(ddl::kConvGemmDgrad);

  // ------------------------------------------------------------------ host runtime
  m.def("driver_available", &ddl::driver_available);
  m.def("plan_buckets",
        [](const std::vector<int64_t>& numels, int64_t first_cap, int64_t cap, int64_t align, int64_t slice) {
          ddl::BucketPlan p = ddl::plan_buckets(numels, first_cap, cap, align, slice);
          py::dict d;
          d["param_bucket"] = p.param_bucket;
          d["param_offset"] = p.param_offset;
          d["bucket_start"] = p.bucket_start;
          d["bucket_numel"] = p.bucket_numel;
          d["bucket_last_param"] = p.bucket_last_param;
          d["bucket_param_count"] = p.bucket_param_count;
          d["total_elems"] = p.total_elems;
          d["hash"] = p.hash;
          return d;
        },
        py::arg("numels"), py::arg("first_cap_elems"), py::arg("cap_elems"), py::arg("align_elems"),
        py::arg("slice_elems"));
  m.def("exchange_fds",
        [](int rank, int world, int fd, const std::string& session, int timeout_ms) {
          py::gil_scoped_release rel;
          return ddl::exchange_fds(rank, world, fd, session, timeout_ms);
        });
  m.def("broadcast_fd", [](int rank, int world, int root, int fd, const std::string& session, int timeout_ms) {
    py::gil_scoped_release rel;
    return ddl::broadcast_fd(rank, world, root, fd, session, timeout_ms);
  });

  py::class_<ddl::SymmArena>(m, "SymmArena")
      .def(py::init<int, int, int, size_t>(), py::arg("rank"), py::arg("world"), py::arg("device"), py::arg("bytes"))
      .def("alloc", &ddl::SymmArena::alloc)
      .def("exchange", &ddl::SymmArena::exchange, py::call_guard<py::gil_scoped_release>())
      .def("multicast_supported", &ddl::SymmArena::multicast_supported)
      .def("mc_create", &ddl::SymmArena::mc_create, py::call_guard<py::gil_scoped_release>())
      .def("mc_bind", &ddl::SymmArena::mc_bind)
      .def("release", &ddl::SymmArena::release)
      .def_property_readonly("bytes", &ddl::SymmArena::bytes)
      .def_property_readonly("local_ptr", &ddl::SymmArena::local_ptr)
      .def_property_readonly("peer_ptrs", &ddl::SymmArena::peer_ptrs)
      .def_property_readonly("mc_ptr", &ddl::SymmArena::mc_ptr)
      .def_property_readonly("last_error", &ddl::SymmArena::last_error);

  // ------------------------------------------------------------------ comm
  py::class_<PyCommCtx>(m, "CommCtx")
      .def(py::init([](const std::vector<uint64_t>& peers, uint64_t mc_base, int rank, int world, uint64_t flag_off,
                       uint64_t grad_off, uint64_t weight_off, uint64_t wbf16_off, uint64_t stage_off,
                       ptr_t epoch_ctr, ptr_t error_flag, uint64_t timeout_ns, uint32_t debug_skew_ns) {
             if (world < 1 || world > ddl::kCommMaxWorld || static_cast<int>(peers.size()) < world)
               throw std::invalid_argument("CommCtx: bad world / peers");
             PyCommCtx x;
             for (int i = 0; i < ddl::kCommMaxWorld; ++i) x.c.peer_base[i] = i < world ? peers[i] : 0;
             x.c.mc_base = mc_base;
             x.c.rank = rank;
             x.c.world = world;
             x.c.flag_off = flag_off;
             x.c.grad_off = grad_off;
             x.c.weight_off = weight_off;
             x.c.wbf16_off = wbf16_off;
             x.c.stage_off = stage_off;
             x.c.epoch_ctr = P<uint32_t>(epoch_ctr);
             x.c.error_flag = P<uint32_t>(error_flag);
             x.c.timeout_ns = timeout_ns;
             x.c.debug_skew_ns = debug_skew_ns;
             return x;
           }),
           py::arg("peers"), py::arg("mc_base"), py::arg("rank"), py::arg("world"), py::arg("flag_off"),
           py::arg("grad_off"), py::arg("weight_off"), py::arg("wbf16_off"), py::arg("stage_off"),
           py::arg("epoch_ctr"), py::arg("error_flag"), py::arg("timeout_ns"), py::arg("debug_skew_ns") = 0)
      .def_property_readonly("has_multicast", [](const PyCommCtx& x) { return x.c.mc_base != 0; });

  m.def("pack_sgd_hyper", [](float lr, float momentum, float dampening, float wd, float grad_scale, bool nesterov,
                             bool first_step) {
    SgdHyper h{lr, momentum, dampening, wd, grad_scale, nesterov ? 1 : 0, first_step ? 1 : 0, 0};
    return py::bytes(reinterpret_cast<const char*>(&h), sizeof(h));
  });
  m.def("fused_sgd_local", [](ptr_t w, ptr_t g, ptr_t mom, ptr_t wb, ptr_t hyper, int64_t numel, int blocks,
                              ptr_t stream) {
    check(ddl::launch_fused_sgd_local(P<float>(w), P<float>(g), P<float>(mom), P<void>(wb), P<const SgdHyper>(hyper),
                                      numel, blocks, S(stream)), "fused_sgd_local");
  });
  m.def("fused_allreduce_sgd", [](const PyCommCtx& c, int64_t start, int64_t numel, ptr_t momentum, ptr_t hyper,
                                  int channel, bool use_mc, bool wire_bf16, int blocks, ptr_t stream,
                                  uint64_t scalar_off, ptr_t scalar_out, bool oneshot, bool closing) {
    BucketArgs b;
    b.oneshot = oneshot ? 1 : 0;
    b.closing = closing ? 1 : 0;
    b.start = start; b.numel = numel; b.momentum = P<float>(momentum); b.hyper = P<const SgdHyper>(hyper);
    b.channel = channel;
    b.scalar_off = scalar_off; b.scalar_out = P<float>(scalar_out);
    check(ddl::launch_fused_allreduce_sgd(c.c, b, use_mc, wire_bf16, blocks, S(stream)), "fused_allreduce_sgd");
  }, py::arg("ctx"), py::arg("start"), py::arg("numel"), py::arg("momentum"), py::arg("hyper"), py::arg("channel"),
     py::arg("use_mc"), py::arg("wire_bf16"), py::arg("blocks"), py::arg("stream"), py::arg("scalar_off") = 0,
     py::arg("scalar_out") = 0, py::arg("oneshot") = false, py::arg("closing") = true);
  m.attr("SCALAR_SLOTS") = ddl::kScalarSlots;

  // ---- native hook -> bucket-launch sequencing (runtime/step_launcher.h) -------------------------------------------------
  m.def("wgrad_note", [](ptr_t side) { ddl::wgrad_note(S(side)); }, "work was enqueued on the weight-gradient side stream");
  m.def("wgrad_join", [](ptr_t consumer) { return ddl::wgrad_join(S(consumer)); },
        "make `consumer` wait for the side-stream work noted since the last join (False: nothing pending)");
  py::class_<ddl::StepLauncher>(m, "StepLauncher")
      .def(py::init([](std::vector<int32_t> param_bucket, std::vector<int32_t> bucket_param_count,
                       std::vector<int64_t> bucket_start, std::vector<int64_t> bucket_numel, const PyCommCtx& ctx, int world,
                       ptr_t W, ptr_t G, ptr_t M, ptr_t Wb, ptr_t hyper_dev, int comm_blocks, int sms, bool use_mc,
                       bool wire_bf16, int64_t oneshot_bytes, uint64_t scalars_off, ptr_t scalars_out, ptr_t comm_stream,
                       py::function stream_fn, py::function hyper_fn) {
             ddl::StepLauncherConfig c;
             c.param_bucket = std::move(param_bucket);
             c.bucket_param_count = std::move(bucket_param_count);
             c.bucket_start = std::move(bucket_start);
             c.bucket_numel = std::move(bucket_numel);
             c.ctx = ctx.c;
             c.world = world;
             c.W = P<float>(W); c.G = P<float>(G); c.M = P<float>(M); c.Wb = P<void>(Wb);
             c.hyper_dev = P<const SgdHyper>(hyper_dev);
             c.comm_blocks = comm_blocks; c.sms = sms; c.use_mc = use_mc; c.wire_bf16 = wire_bf16;
             c.oneshot_bytes = oneshot_bytes; c.scalars_off = scalars_off; c.scalars_out = P<float>(scalars_out);
             c.comm_stream = S(comm_stream);
             return new ddl::StepLauncher(
                 std::move(c), [stream_fn]() { return S(stream_fn().cast<ptr_t>()); },
                 [hyper_fn](cudaStream_t st) { hyper_fn(reinterpret_cast<ptr_t>(st)); });
           }),
           py::arg("param_bucket"), py::arg("bucket_param_count"), py::arg("bucket_start"), py::arg("bucket_numel"),
           py::arg("ctx"), py::arg("world"), py::arg("W"), py::arg("G"), py::arg("M"), py::arg("Wb"), py::arg("hyper_dev"),
           py::arg("comm_blocks"), py::arg("sms"), py::arg("use_mc"), py::arg("wire_bf16"), py::arg("oneshot_bytes"),
           py::arg("scalars_off"), py::arg("scalars_out"), py::arg("comm_stream"), py::arg("stream_fn"), py::arg("hyper_fn"))
      .def("on_ready", &ddl::StepLauncher::on_ready)
      .def("hook", [](ddl::StepLauncher& s, int idx) {
             // the autograd hook itself: a C++ callable (called as hook(param)); no Python frame on the per-parameter path
             return py::cpp_function([&s, idx](py::args) { s.on_ready(idx); });
           }, py::keep_alive<0, 1>())
      .def("finish", &ddl::StepLauncher::finish)
      .def("reset", &ddl::StepLauncher::reset)
      .def("set_hold", &ddl::StepLauncher::set_hold)
      .def("set_scalars_pending", &ddl::StepLauncher::set_scalars_pending)
      .def_property_readonly("next_bucket", &ddl::StepLauncher::next_bucket)
      .def_property_readonly("launches", &ddl::StepLauncher::launches);
  m.def("allreduce", [](const PyCommCtx& c, int channel, uint64_t off, int64_t numel, bool bf16, float scale,
                        bool use_mc, bool oneshot, int blocks, ptr_t stream) {
    check(ddl::launch_allreduce(c.c, channel, off, numel, bf16, scale, use_mc, oneshot, blocks, S(stream)), "allreduce");
  });
  m.def("broadcast", [](const PyCommCtx& c, int channel, uint64_t off, int64_t bytes, int root, bool use_mc,
                        int blocks, ptr_t stream) {
    check(ddl::launch_broadcast(c.c, channel, off, bytes, root, use_mc, blocks, S(stream)), "broadcast");
  });
  m.def("barrier", [](const PyCommCtx& c, int channel, ptr_t stream) {
    check(ddl::launch_barrier(c.c, channel, S(stream)), "barrier");
  });
  m.def("allgather_slices", [](const PyCommCtx& c, int channel, ptr_t src, uint64_t dst_off, int64_t start,
                               int64_t numel, bool use_mc, int blocks, ptr_t stream) {
    check(ddl::launch_allgather_slices(c.c, channel, P<const float>(src), dst_off, start, numel, use_mc, blocks,
                                       S(stream)), "allgather_slices");
  });

  // ------------------------------------------------------------------ conv / GEMM
  m.def("conv_timeout_info", []() {
    unsigned int v[8];
    check(ddl::conv_timeout_info(v), "conv_timeout_info");
    return std::vector<unsigned int>(v, v + 8);
  }, "post-mortem of the first timed-out mbarrier wait (flag, site, block, thread, parity); clears the record");
  m.def("set_conv_wait_hint", &ddl::set_conv_wait_hint, "tuning hook: suspend-time hint (ns) of the conv kernels' mbarrier waits, 0 = none");
  m.def("set_bn_reverse", &ddl::set_bn_reverse, "1 (default) = BN forward / backward-reduce walk the rows from the end (L2 reuse of the producer's tail), 0 = front to back");
  m.def("set_pdl", &ddl::set_pdl, "0 = plain stream order, 1 = conv / BN kernels allow programmatic dependent launch (default), 2 = + trigger at the last tile, 3 = + trigger at block start");
  m.def("set_conv_persistent", &ddl::set_conv_persistent, "tuning hook: 0 = never the persistent conv kernel, 1 = policy, 2 = always");
  m.def("set_conv_cluster", &ddl::set_conv_cluster, "tuning hook: 1 = the persistent kernel runs as CTA pairs sharing the weight tile by TMA multicast");
  m.def("set_conv_deep", &ddl::set_conv_deep, "tuning hook: 2 = persistent CTA pairs wherever they apply, 3/4 = persistent single CTAs");
  m.def("set_wgrad_swap", &ddl::set_wgrad_swap, "tuning hook: 0 = no operand-role swap for narrow-output wgrad tiles");
  m.def("set_conv_force_stages", &ddl::set_conv_force_stages, "tuning hook: force the pipeline depth (0 = policy)");
  m.def("conv_gemm",
        [](int mode, ptr_t src, ptr_t out, ptr_t add, ptr_t bias, ptr_t sum, ptr_t sumsq, int M, int KB, int ldc,
           int srcH, int srcW, int srcC, int dstH, int dstW, int R, int Sx, int stride, int pad, int dil,
           int cchunks, int relu, int n_valid, ptr_t w, int w_rows, int w_cols, int n_total, ptr_t a_matrix, int a_cols,
           int batch, int tw, int th, int tn, int zfill, ptr_t stream, int pad_w, int kstride, ptr_t add_mask,
           ptr_t bnr_y, ptr_t bnr_gamma, ptr_t bnr_beta, ptr_t bnr_mean, ptr_t bnr_invstd, int variant, int fp8,
           ptr_t deq_a, ptr_t deq_b, ptr_t sfa, ptr_t sfb, ptr_t bnr_mask, int grouped) {
          ConvArgs a;
          a.grouped = grouped;
          a.variant = variant;
          a.fp8 = fp8; a.deq_a = P<const float>(deq_a); a.deq_b = P<const float>(deq_b);
          a.sfa = P<const uint8_t>(sfa); a.sfb = P<const uint8_t>(sfb);
          a.bnr_y = P<const __nv_bfloat16>(bnr_y); a.bnr_gamma = P<const float>(bnr_gamma);
          a.bnr_beta = P<const float>(bnr_beta); a.bnr_mean = P<const float>(bnr_mean);
          a.bnr_invstd = P<const float>(bnr_invstd); a.bnr_mask = P<const uint8_t>(bnr_mask);
          a.add_mask = P<const uint8_t>(add_mask);
          a.zfill = zfill;
          a.pad_w = pad_w < 0 ? pad : pad_w;
          a.kstride = kstride > 0 ? kstride : cchunks * 64;
          a.src = P<const __nv_bfloat16>(src); a.out = P<__nv_bfloat16>(out); a.add = P<const __nv_bfloat16>(add);
          a.bias = P<const float>(bias); a.sum = P<float>(sum); a.sumsq = P<float>(sumsq);
          a.M = M; a.KB = KB; a.ldc = ldc; a.srcH = srcH; a.srcW = srcW; a.srcC = srcC; a.dstH = dstH; a.dstW = dstW;
          a.R = R; a.S = Sx; a.stride = stride; a.pad = pad; a.dil = dil; a.cchunks = cchunks; a.relu = relu; a.n_valid = n_valid;
          a.stages = 0; a.batch = batch; a.tw = tw; a.th = th; a.tn = tn; a.tiles_w = 0; a.tiles_h = 0;
          check(ddl::launch_conv_gemm(mode, a, P<const void>(w), w_rows, w_cols, n_total, P<const void>(a_matrix),
                                      a_cols, S(stream)), "conv_gemm");
        },
        py::arg("mode"), py::arg("src"), py::arg("out"), py::arg("add"), py::arg("bias"), py::arg("sum"), py::arg("sumsq"),
        py::arg("M"), py::arg("KB"), py::arg("ldc"), py::arg("srcH"), py::arg("srcW"), py::arg("srcC"), py::arg("dstH"),
        py::arg("dstW"), py::arg("R"), py::arg("S"), py::arg("stride"), py::arg("pad"), py::arg("dil"), py::arg("cchunks"),
        py::arg("relu"), py::arg("n_valid"), py::arg("w"), py::arg("w_rows"), py::arg("w_cols"), py::arg("n_total"),
        py::arg("a_matrix"), py::arg("a_cols"), py::arg("batch"), py::arg("tw"), py::arg("th"), py::arg("tn"),
        py::arg("zfill"), py::arg("stream"), py::arg("pad_w") = -1, py::arg("kstride") = 0, py::arg("add_mask") = 0,
        py::arg("bnr_y") = 0, py::arg("bnr_gamma") = 0, py::arg("bnr_beta") = 0, py::arg("bnr_mean") = 0,
        py::arg("bnr_invstd") = 0, py::arg("variant") = 0, py::arg("fp8") = 0, py::arg("deq_a") = 0,
        py::arg("deq_b") = 0, py::arg("sfa") = 0, py::arg("sfb") = 0, py::arg("bnr_mask") = 0, py::arg("grouped") = 0);
  m.def("conv_wgrad",
        [](int mode, ptr_t x, ptr_t dy, ptr_t dw, int M, int Cout, int dy_ld, int ldw, int ncols, int H, int W, int C, int Pq,
           int Q, int R, int Sx, int stride, int pad, int dil, int cchunks, int splits, int batch, int tw, int th, int tn,
           ptr_t stream, int pad_w, int Cpad, int Cw, int group_width) {
          WgradArgs a;
          a.group_width = group_width;
          a.pad_w = pad_w < 0 ? pad : pad_w;
          a.Cpad = Cpad > 0 ? Cpad : ncols;      // default: one tap spanning every column (stem scratch, GEMM)
          a.Cw = Cw > 0 ? Cw : ncols;
          a.stages = 0; a.batch = batch; a.tw = tw; a.th = th; a.tn = tn; a.tiles_w = 0; a.tiles_h = 0;
          a.x = P<const __nv_bfloat16>(x); a.dw = P<float>(dw); a.M = M; a.Cout = Cout; a.dy_ld = dy_ld; a.ldw = ldw; a.ncols = ncols;
          a.H = H; a.W = W; a.C = C; a.P = Pq; a.Q = Q; a.R = R; a.S = Sx; a.stride = stride; a.pad = pad; a.dil = dil;
          a.cchunks = cchunks; a.kb_per_split = 0; a.total_kb = 0; a.mode = mode;
          check(ddl::launch_conv_wgrad(a, P<const void>(dy), P<const void>(x), splits, S(stream)), "conv_wgrad");
        },
        py::arg("mode"), py::arg("x"), py::arg("dy"), py::arg("dw"), py::arg("M"), py::arg("Cout"), py::arg("dy_ld"),
        py::arg("ldw"), py::arg("ncols"), py::arg("H"), py::arg("W"), py::arg("C"), py::arg("P"), py::arg("Q"), py::arg("R"),
        py::arg("S"), py::arg("stride"), py::arg("pad"), py::arg("dil"), py::arg("cchunks"), py::arg("splits"),
        py::arg("batch"), py::arg("tw"), py::arg("th"), py::arg("tn"), py::arg("stream"), py::arg("pad_w") = -1,
        py::arg("Cpad") = 0, py::arg("Cw") = 0, py::arg("group_width") = 0);
  m.def("expand_grouped_weight", [](ptr_t w, ptr_t out, int cout, int taps, int gw, ptr_t stream) {
    check(ddl::launch_expand_grouped_weight(P<const void>(w), P<void>(out), cout, taps, gw, S(stream)),
          "expand_grouped_weight");
  }, "compact grouped conv weights [Cout][taps*gw] bf16 -> block-diagonal [Cout][taps*64] (zeros off the group)");

  // ------------------------------------------------------------------ BN / activation
  m.def("bn_act_fwd", [](ptr_t x, ptr_t residual, ptr_t z, ptr_t sum, ptr_t sumsq, ptr_t gamma, ptr_t beta,
                         ptr_t mean, ptr_t invstd, ptr_t rmean, ptr_t rvar, float eps, float momentum, int M, int C,
                         int relu, bool train, int sms, ptr_t stream, ptr_t mask, ptr_t zq, ptr_t zq_slot,
                         ptr_t sample_scale, int hw) {
    BnFwdArgs a{};
    a.mask = P<uint8_t>(mask);
    a.sample_scale = P<const float>(sample_scale); a.hw = hw;
    a.zq = P<uint8_t>(zq); a.zq_slot = P<ddl::Fp8Slot>(zq_slot);
    a.x = P<const __nv_bfloat16>(x); a.residual = P<const __nv_bfloat16>(residual); a.z = P<__nv_bfloat16>(z);
    a.sum = P<const float>(sum); a.sumsq = P<const float>(sumsq); a.gamma = P<const float>(gamma);
    a.beta = P<const float>(beta); a.mean = P<float>(mean); a.invstd = P<float>(invstd);
    a.running_mean = P<float>(rmean); a.running_var = P<float>(rvar); a.eps = eps; a.momentum = momentum;
    a.M = M; a.C = C; a.relu = relu;
    check(ddl::launch_bn_act_fwd(a, train, sms, S(stream)), "bn_act_fwd");
  }, py::arg("x"), py::arg("residual"), py::arg("z"), py::arg("sum"), py::arg("sumsq"), py::arg("gamma"), py::arg("beta"),
     py::arg("mean"), py::arg("invstd"), py::arg("rmean"), py::arg("rvar"), py::arg("eps"), py::arg("momentum"),
     py::arg("M"), py::arg("C"), py::arg("relu"), py::arg("train"), py::arg("sms"), py::arg("stream"), py::arg("mask") = 0,
     py::arg("zq") = 0, py::arg("zq_slot") = 0, py::arg("sample_scale") = 0, py::arg("hw") = 0);
  m.def("bn_act_bwd", [](ptr_t dz, ptr_t z, ptr_t x, ptr_t dx, ptr_t dres, ptr_t mean, ptr_t invstd, ptr_t gamma,
                         ptr_t beta, ptr_t dgamma, ptr_t dbeta, ptr_t gamma_grad, ptr_t beta_grad, int M, int C,
                         int relu, int mask_from_x, int sms, ptr_t stream, ptr_t zmask, bool skip_reduce, ptr_t dxq,
                         ptr_t dxq_slot, ptr_t sample_scale, int hw) {
    BnBwdArgs a{};
    a.zmask = P<const uint8_t>(zmask);
    a.sample_scale = P<const float>(sample_scale); a.hw = hw;
    a.dxq = P<uint8_t>(dxq); a.dxq_slot = P<ddl::Fp8Slot>(dxq_slot);
    a.dz = P<const __nv_bfloat16>(dz); a.z = P<const __nv_bfloat16>(z); a.x = P<const __nv_bfloat16>(x);
    a.dx = P<__nv_bfloat16>(dx); a.dres = P<__nv_bfloat16>(dres); a.mean = P<const float>(mean);
    a.invstd = P<const float>(invstd); a.gamma = P<const float>(gamma); a.dgamma = P<float>(dgamma);
    a.dbeta = P<float>(dbeta); a.gamma_grad = P<float>(gamma_grad); a.beta_grad = P<float>(beta_grad);
    a.M = M; a.C = C; a.relu = relu; a.beta = P<const float>(beta); a.mask_from_x = mask_from_x;
    check(ddl::launch_bn_act_bwd(a, sms, S(stream), skip_reduce), "bn_act_bwd");
  }, py::arg("dz"), py::arg("z"), py::arg("x"), py::arg("dx"), py::arg("dres"), py::arg("mean"), py::arg("invstd"),
     py::arg("gamma"), py::arg("beta"), py::arg("dgamma"), py::arg("dbeta"), py::arg("gamma_grad"), py::arg("beta_grad"),
     py::arg("M"), py::arg("C"), py::arg("relu"), py::arg("mask_from_x"), py::arg("sms"), py::arg("stream"),
     py::arg("zmask") = 0, py::arg("skip_reduce") = false, py::arg("dxq") = 0, py::arg("dxq_slot") = 0,
     py::arg("sample_scale") = 0, py::arg("hw") = 0);
  m.def("bn_relu_maxpool_fwd", [](ptr_t x, ptr_t pooled, ptr_t argmax, ptr_t sum, ptr_t sumsq, ptr_t gamma, ptr_t beta,
                                  ptr_t mean, ptr_t invstd, ptr_t rmean, ptr_t rvar, float eps, float momentum, int N, int H,
                                  int W, int C, int Pq, int Q, int k, int stride, int pad, int sms, ptr_t stream) {
    BnFwdArgs a{};
    a.x = P<const __nv_bfloat16>(x); a.residual = nullptr; a.z = nullptr; a.mask = nullptr;
    a.sum = P<const float>(sum); a.sumsq = P<const float>(sumsq); a.gamma = P<const float>(gamma);
    a.beta = P<const float>(beta); a.mean = P<float>(mean); a.invstd = P<float>(invstd);
    a.running_mean = P<float>(rmean); a.running_var = P<float>(rvar); a.eps = eps; a.momentum = momentum;
    a.M = N * H * W; a.C = C; a.relu = 1;
    check(ddl::launch_bn_relu_maxpool_fwd(a, pool_args(N, H, W, C, Pq, Q, k, stride, pad), P<__nv_bfloat16>(pooled),
                                          P<uint8_t>(argmax), sms, S(stream)), "bn_relu_maxpool_fwd");
  });
  m.def("bn_pool_bwd", [](ptr_t dy_pooled, ptr_t argmax, ptr_t x, ptr_t dx, ptr_t mean, ptr_t invstd, ptr_t gamma, ptr_t beta,
                          ptr_t dgamma, ptr_t dbeta, ptr_t gamma_grad, ptr_t beta_grad, int N, int H, int W, int C, int Pq,
                          int Q, int k, int stride, int pad, int sms, ptr_t stream) {
    BnBwdArgs a{};
    a.dz = nullptr; a.z = nullptr; a.x = P<const __nv_bfloat16>(x); a.dx = P<__nv_bfloat16>(dx); a.dres = nullptr;
    a.mean = P<const float>(mean); a.invstd = P<const float>(invstd); a.gamma = P<const float>(gamma);
    a.beta = P<const float>(beta); a.dgamma = P<float>(dgamma); a.dbeta = P<float>(dbeta);
    a.gamma_grad = P<float>(gamma_grad); a.beta_grad = P<float>(beta_grad); a.M = N * H * W; a.C = C; a.relu = 1;
    a.mask_from_x = 1; a.zmask = nullptr;
    check(ddl::launch_bn_pool_bwd(a, pool_args(N, H, W, C, Pq, Q, k, stride, pad), P<const __nv_bfloat16>(dy_pooled),
                                  P<const uint8_t>(argmax), sms, S(stream)), "bn_pool_bwd");
  });
  // ------------------------------------------------------------------ depthwise 3x3 convolution
  // k: the kernel size, 3 (padding 1, depthwise.cu) or 5 (padding 2, depthwise5.cu)
  m.def("dwconv_fwd", [](ptr_t x, ptr_t w, ptr_t y, ptr_t sum, ptr_t sumsq, int N, int H, int W, int C, int Pq, int Q,
                         int stride, int sms, ptr_t stream, int k) {
    ddl::DwConvArgs a{};
    a.x = P<const __nv_bfloat16>(x); a.w = P<const __nv_bfloat16>(w); a.y = P<__nv_bfloat16>(y);
    a.sum = P<float>(sum); a.sumsq = P<float>(sumsq);
    a.N = N; a.H = H; a.W = W; a.C = C; a.P = Pq; a.Q = Q; a.stride = stride;
    check(k == 3 ? ddl::launch_dwconv_fwd(a, sms, S(stream))
                 : k == 5 ? ddl::launch_dwconv5_fwd(a, sms, S(stream)) : cudaErrorInvalidValue, "dwconv_fwd");
  }, py::arg("x"), py::arg("w"), py::arg("y"), py::arg("sum"), py::arg("sumsq"), py::arg("N"), py::arg("H"), py::arg("W"),
     py::arg("C"), py::arg("P"), py::arg("Q"), py::arg("stride"), py::arg("sms"), py::arg("stream"), py::arg("k") = 3);
  m.def("dwconv_dgrad", [](ptr_t dy, ptr_t w, ptr_t dx, int N, int H, int W, int C, int Pq, int Q, int stride, int sms,
                           ptr_t stream, int k) {
    ddl::DwConvArgs a{};
    a.dy = P<const __nv_bfloat16>(dy); a.w = P<const __nv_bfloat16>(w); a.y = P<__nv_bfloat16>(dx);
    a.N = N; a.H = H; a.W = W; a.C = C; a.P = Pq; a.Q = Q; a.stride = stride;
    check(k == 3 ? ddl::launch_dwconv_dgrad(a, sms, S(stream))
                 : k == 5 ? ddl::launch_dwconv5_dgrad(a, sms, S(stream)) : cudaErrorInvalidValue, "dwconv_dgrad");
  }, py::arg("dy"), py::arg("w"), py::arg("dx"), py::arg("N"), py::arg("H"), py::arg("W"), py::arg("C"), py::arg("P"),
     py::arg("Q"), py::arg("stride"), py::arg("sms"), py::arg("stream"), py::arg("k") = 3);
  m.def("dwconv_wgrad", [](ptr_t x, ptr_t dy, ptr_t gw, int N, int H, int W, int C, int Pq, int Q, int stride, int sms,
                           ptr_t stream, int k) {
    ddl::DwConvArgs a{};
    a.x = P<const __nv_bfloat16>(x); a.dy = P<const __nv_bfloat16>(dy); a.gw = P<float>(gw);
    a.N = N; a.H = H; a.W = W; a.C = C; a.P = Pq; a.Q = Q; a.stride = stride;
    check(k == 3 ? ddl::launch_dwconv_wgrad(a, sms, S(stream))
                 : k == 5 ? ddl::launch_dwconv5_wgrad(a, sms, S(stream)) : cudaErrorInvalidValue, "dwconv_wgrad");
  }, py::arg("x"), py::arg("dy"), py::arg("gw"), py::arg("N"), py::arg("H"), py::arg("W"), py::arg("C"), py::arg("P"),
     py::arg("Q"), py::arg("stride"), py::arg("sms"), py::arg("stream"), py::arg("k") = 3);
  // ------------------------------------------------------------------ depthwise 7x7 with a bias (ConvNeXt)
  // l1: the L1 mapping instead of the halo tile (tools/depthwise_bench.py compares the two)
  m.def("dwconv7_fwd", [](ptr_t x, ptr_t w, ptr_t bias, ptr_t y, int N, int H, int W, int C, int sms, ptr_t stream,
                          int l1) {
    ddl::Dw7Args a{};
    a.x = P<const __nv_bfloat16>(x); a.w = P<const __nv_bfloat16>(w); a.bias = P<const float>(bias);
    a.y = P<__nv_bfloat16>(y); a.N = N; a.H = H; a.W = W; a.C = C;
    check(ddl::launch_dwconv7_fwd(a, sms, l1 != 0, S(stream)), "dwconv7_fwd");
  }, py::arg("x"), py::arg("w"), py::arg("bias"), py::arg("y"), py::arg("N"), py::arg("H"), py::arg("W"), py::arg("C"),
     py::arg("sms"), py::arg("stream"), py::arg("l1") = 0);
  m.def("dwconv7_dgrad", [](ptr_t dy, ptr_t w, ptr_t add, ptr_t dx, int N, int H, int W, int C, int sms, ptr_t stream,
                            int l1) {
    ddl::Dw7Args a{};
    a.dy = P<const __nv_bfloat16>(dy); a.w = P<const __nv_bfloat16>(w); a.add = P<const __nv_bfloat16>(add);
    a.y = P<__nv_bfloat16>(dx); a.N = N; a.H = H; a.W = W; a.C = C;
    check(ddl::launch_dwconv7_dgrad(a, sms, l1 != 0, S(stream)), "dwconv7_dgrad");
  }, py::arg("dy"), py::arg("w"), py::arg("add"), py::arg("dx"), py::arg("N"), py::arg("H"), py::arg("W"), py::arg("C"),
     py::arg("sms"), py::arg("stream"), py::arg("l1") = 0);
  m.def("dwconv7_wgrad", [](ptr_t x, ptr_t dy, ptr_t gw, ptr_t gb, int N, int H, int W, int C, int sms, ptr_t stream) {
    ddl::Dw7Args a{};
    a.x = P<const __nv_bfloat16>(x); a.dy = P<const __nv_bfloat16>(dy); a.gw = P<float>(gw); a.gb = P<float>(gb);
    a.N = N; a.H = H; a.W = W; a.C = C;
    check(ddl::launch_dwconv7_wgrad(a, sms, S(stream)), "dwconv7_wgrad");
  });
  // ------------------------------------------------------------------ ConvNeXt row kernels (LayerNorm, GELU, layer scale)
  m.def("layer_norm_fwd", [](ptr_t x, ptr_t gamma, ptr_t beta, ptr_t y, ptr_t mean, ptr_t rstd, int M, int C, float eps,
                             int sms, ptr_t stream) {
    check(ddl::launch_layer_norm_fwd(P<const __nv_bfloat16>(x), P<const float>(gamma), P<const float>(beta),
                                     P<__nv_bfloat16>(y), P<float>(mean), P<float>(rstd), M, C, eps, sms, S(stream)),
          "layer_norm_fwd");
  });
  m.def("layer_norm_bwd", [](ptr_t dy, ptr_t x, ptr_t mean, ptr_t rstd, ptr_t gamma, ptr_t dx, ptr_t dgamma, ptr_t dbeta,
                             int M, int C, int sms, ptr_t stream) {
    check(ddl::launch_layer_norm_bwd(P<const __nv_bfloat16>(dy), P<const __nv_bfloat16>(x), P<const float>(mean),
                                     P<const float>(rstd), P<const float>(gamma), P<__nv_bfloat16>(dx), P<float>(dgamma),
                                     P<float>(dbeta), M, C, sms, S(stream)), "layer_norm_bwd");
  });
  m.def("gelu_fwd", [](ptr_t h, ptr_t g, int64_t n, int sms, ptr_t stream) {
    check(ddl::launch_gelu_fwd(P<const __nv_bfloat16>(h), P<__nv_bfloat16>(g), n, sms, S(stream)), "gelu_fwd");
  });
  m.def("gelu_bwd", [](ptr_t dg, ptr_t h, ptr_t dh, ptr_t dbias, int M, int C, int sms, ptr_t stream) {
    check(ddl::launch_gelu_bwd(P<const __nv_bfloat16>(dg), P<const __nv_bfloat16>(h), P<__nv_bfloat16>(dh), P<float>(dbias),
                               M, C, sms, S(stream)), "gelu_bwd");
  });
  m.def("layer_scale_fwd", [](ptr_t y, ptr_t ls, ptr_t keep, ptr_t x, ptr_t z, int M, int C, int hw, int sms,
                              ptr_t stream) {
    check(ddl::launch_layer_scale_fwd(P<const __nv_bfloat16>(y), P<const float>(ls), P<const float>(keep),
                                      P<const __nv_bfloat16>(x), P<__nv_bfloat16>(z), M, C, hw, sms, S(stream)),
          "layer_scale_fwd");
  });
  m.def("layer_scale_bwd", [](ptr_t dz, ptr_t y, ptr_t ls, ptr_t keep, ptr_t dy, ptr_t dls, ptr_t dbias, int M, int C,
                              int hw, int sms, ptr_t stream) {
    check(ddl::launch_layer_scale_bwd(P<const __nv_bfloat16>(dz), P<const __nv_bfloat16>(y), P<const float>(ls),
                                      P<const float>(keep), P<__nv_bfloat16>(dy), P<float>(dls), P<float>(dbias), M, C, hw,
                                      sms, S(stream)), "layer_scale_bwd");
  });
  // ------------------------------------------------------------------ ViT: attention and row kernels
  m.def("attention_fwd", [](ptr_t qkv, ptr_t o, ptr_t lse, int N, int L, int H, int C, ptr_t stream) {
    check(ddl::launch_attention_fwd(P<const __nv_bfloat16>(qkv), P<__nv_bfloat16>(o), P<float>(lse), N, L, H, C,
                                    S(stream)), "attention_fwd");
  });
  m.def("attention_bwd", [](ptr_t qkv, ptr_t o, ptr_t dout, ptr_t lse, ptr_t delta, ptr_t dqkv, int N, int L, int H,
                            int C, ptr_t stream) {
    check(ddl::launch_attention_bwd(P<const __nv_bfloat16>(qkv), P<const __nv_bfloat16>(o), P<const __nv_bfloat16>(dout),
                                    P<const float>(lse), P<float>(delta), P<__nv_bfloat16>(dqkv), N, L, H, C, S(stream)),
          "attention_bwd");
  });
  m.def("add_layer_norm_fwd", [](ptr_t x, ptr_t add, ptr_t gamma, ptr_t beta, ptr_t x1, ptr_t y, ptr_t mean, ptr_t rstd,
                                 int M, int C, float eps, int sms, ptr_t stream) {
    check(ddl::launch_add_layer_norm_fwd(P<const __nv_bfloat16>(x), P<const __nv_bfloat16>(add), P<const float>(gamma),
                                         P<const float>(beta), P<__nv_bfloat16>(x1), P<__nv_bfloat16>(y), P<float>(mean),
                                         P<float>(rstd), M, C, eps, sms, S(stream)), "add_layer_norm_fwd");
  });
  m.def("layer_norm_bwd_add", [](ptr_t dy, ptr_t x, ptr_t mean, ptr_t rstd, ptr_t gamma, ptr_t dres, ptr_t dx,
                                 ptr_t dgamma, ptr_t dbeta, int M, int C, int sms, ptr_t stream) {
    check(ddl::launch_layer_norm_bwd_add(P<const __nv_bfloat16>(dy), P<const __nv_bfloat16>(x), P<const float>(mean),
                                         P<const float>(rstd), P<const float>(gamma), P<const __nv_bfloat16>(dres),
                                         P<__nv_bfloat16>(dx), P<float>(dgamma), P<float>(dbeta), M, C, sms, S(stream)),
          "layer_norm_bwd_add");
  });
  m.def("patchify", [](ptr_t img, ptr_t out, int N, int H, int W, int P_, int sms, ptr_t stream) {
    check(ddl::launch_patchify(P<const __nv_bfloat16>(img), P<__nv_bfloat16>(out), N, H, W, P_, sms, S(stream)),
          "patchify");
  });
  m.def("tokens_fwd", [](ptr_t patch, ptr_t cls, ptr_t pos, ptr_t tok, int N, int L, int C, int sms, ptr_t stream) {
    check(ddl::launch_tokens_fwd(P<const __nv_bfloat16>(patch), P<const float>(cls), P<const float>(pos),
                                 P<__nv_bfloat16>(tok), N, L, C, sms, S(stream)), "tokens_fwd");
  });
  m.def("tokens_bwd", [](ptr_t dtok, ptr_t dpatch, ptr_t colsum, ptr_t dpos, ptr_t dcls, ptr_t dbias, int N, int L, int C,
                         ptr_t stream) {
    check(ddl::launch_tokens_bwd(P<const __nv_bfloat16>(dtok), P<__nv_bfloat16>(dpatch), P<float>(colsum), P<float>(dpos),
                                 P<float>(dcls), P<float>(dbias), N, L, C, S(stream)), "tokens_bwd");
  });
  // ------------------------------------------------------------------ Swin: window attention and patch merging
  m.def("window_attention_fwd", [](ptr_t qkv, ptr_t table, ptr_t o, ptr_t lse, int N, int H, int W, int heads, int C,
                                   int sy, int sx, ptr_t stream) {
    check(ddl::launch_window_attention_fwd(P<const __nv_bfloat16>(qkv), P<const float>(table), P<__nv_bfloat16>(o),
                                           P<float>(lse), N, H, W, heads, C, sy, sx, S(stream)), "window_attention_fwd");
  });
  m.def("window_attention_bwd", [](ptr_t qkv, ptr_t table, ptr_t o, ptr_t dout, ptr_t lse, ptr_t dqkv, ptr_t dtable,
                                   ptr_t scratch, int N, int H, int W, int heads, int C, int sy, int sx, ptr_t stream) {
    check(ddl::launch_window_attention_bwd(P<const __nv_bfloat16>(qkv), P<const float>(table),
                                           P<const __nv_bfloat16>(o), P<const __nv_bfloat16>(dout), P<const float>(lse),
                                           P<__nv_bfloat16>(dqkv), P<float>(dtable), P<float>(scratch), N, H, W, heads, C,
                                           sy, sx, S(stream)), "window_attention_bwd");
  });
  m.def("window_attention_bwd_scratch_floats", [](int N, int H, int heads) {
    return ddl::window_attention_bwd_scratch_floats(N, H, heads);
  });
  // ------------------------------------------------------------------ MaxViT: partition (grid / window) attention
  m.def("grid_attention_fwd", [](ptr_t qkv, ptr_t table, ptr_t o, ptr_t lse, int N, int H, int W, int heads, int C,
                                 bool grid, float scale, ptr_t stream) {
    check(ddl::launch_grid_attention_fwd(P<const __nv_bfloat16>(qkv), P<const float>(table), P<__nv_bfloat16>(o),
                                         P<float>(lse), N, H, W, heads, C, grid, scale, S(stream)), "grid_attention_fwd");
  });
  m.def("grid_attention_bwd", [](ptr_t qkv, ptr_t table, ptr_t o, ptr_t dout, ptr_t lse, ptr_t dqkv, ptr_t dtable,
                                 ptr_t scratch, int N, int H, int W, int heads, int C, bool grid, float scale,
                                 ptr_t stream) {
    check(ddl::launch_grid_attention_bwd(P<const __nv_bfloat16>(qkv), P<const float>(table), P<const __nv_bfloat16>(o),
                                         P<const __nv_bfloat16>(dout), P<const float>(lse), P<__nv_bfloat16>(dqkv),
                                         P<float>(dtable), P<float>(scratch), N, H, W, heads, C, grid, scale,
                                         S(stream)), "grid_attention_bwd");
  });
  m.def("grid_attention_bwd_scratch_floats", [](int N, int H, int heads) {
    return ddl::grid_attention_bwd_scratch_floats(N, H, heads);
  });
  m.def("patch_merge_fwd", [](ptr_t x, ptr_t gamma, ptr_t beta, ptr_t y, ptr_t mean, ptr_t rstd, int N, int H, int W,
                              int C, float eps, int sms, ptr_t stream) {
    check(ddl::launch_patch_merge_fwd(P<const __nv_bfloat16>(x), P<const float>(gamma), P<const float>(beta),
                                      P<__nv_bfloat16>(y), P<float>(mean), P<float>(rstd), N, H, W, C, eps, sms,
                                      S(stream)), "patch_merge_fwd");
  });
  m.def("patch_merge_bwd", [](ptr_t dy, ptr_t x, ptr_t mean, ptr_t rstd, ptr_t gamma, ptr_t dx, ptr_t dgamma,
                              ptr_t dbeta, ptr_t scratch, int N, int H, int W, int C, int sms, ptr_t stream) {
    check(ddl::launch_patch_merge_bwd(P<const __nv_bfloat16>(dy), P<const __nv_bfloat16>(x), P<const float>(mean),
                                      P<const float>(rstd), P<const float>(gamma), P<__nv_bfloat16>(dx), P<float>(dgamma),
                                      P<float>(dbeta), P<float>(scratch), N, H, W, C, sms, S(stream)),
          "patch_merge_bwd");
  });
  m.def("patch_merge_bwd_blocks", [](int sms) { return ddl::patch_merge_bwd_blocks(sms); });
  // ------------------------------------------------------------------ Swin V2: cosine window attention, CPB, merge gather
  m.def("window_attention_v2_fwd", [](ptr_t qkv, ptr_t table, ptr_t scale, ptr_t qb, ptr_t vb, ptr_t o, ptr_t lse, int N,
                                      int H, int W, int heads, int C, int sy, int sx, ptr_t stream) {
    check(ddl::launch_window_attention_v2_fwd(P<const __nv_bfloat16>(qkv), P<const float>(table), P<const float>(scale),
                                              P<const float>(qb), P<const float>(vb), P<__nv_bfloat16>(o), P<float>(lse),
                                              N, H, W, heads, C, sy, sx, S(stream)), "window_attention_v2_fwd");
  });
  m.def("window_attention_v2_bwd", [](ptr_t qkv, ptr_t table, ptr_t scale, ptr_t qb, ptr_t vb, ptr_t o, ptr_t dout,
                                      ptr_t lse, ptr_t dqkv, ptr_t dtable, ptr_t dscale, ptr_t dbias, ptr_t scratch, int N,
                                      int H, int W, int heads, int C, int sy, int sx, bool bias_pad_only,
                                      ptr_t stream) {
    check(ddl::launch_window_attention_v2_bwd(P<const __nv_bfloat16>(qkv), P<const float>(table), P<const float>(scale),
                                              P<const float>(qb), P<const float>(vb), P<const __nv_bfloat16>(o),
                                              P<const __nv_bfloat16>(dout), P<const float>(lse), P<__nv_bfloat16>(dqkv),
                                              P<float>(dtable), P<float>(dscale), P<float>(dbias), P<float>(scratch), N, H,
                                              W, heads, C, sy, sx, bias_pad_only, S(stream)),
          "window_attention_v2_bwd");
  });
  m.def("window_attention_v2_bwd_scratch_floats", [](int N, int H, int heads) {
    return ddl::window_attention_v2_bwd_scratch_floats(N, H, heads);
  });
  m.def("cpb_fwd", [](ptr_t coords, ptr_t w1, ptr_t b1, ptr_t w2, ptr_t table, ptr_t qkv_b, ptr_t qkv_b_eff, int heads,
                      int C, ptr_t stream) {
    check(ddl::launch_cpb_fwd(P<const float>(coords), P<const float>(w1), P<const float>(b1), P<const float>(w2),
                              P<float>(table), P<const float>(qkv_b), P<float>(qkv_b_eff), heads, C, S(stream)), "cpb_fwd");
  });
  m.def("cpb_bwd", [](ptr_t coords, ptr_t w1, ptr_t b1, ptr_t w2, ptr_t table, ptr_t dtable, ptr_t dw1, ptr_t db1,
                      ptr_t dw2, ptr_t scratch, int heads, ptr_t stream) {
    check(ddl::launch_cpb_bwd(P<const float>(coords), P<const float>(w1), P<const float>(b1), P<const float>(w2),
                              P<const float>(table), P<const float>(dtable), P<float>(dw1), P<float>(db1), P<float>(dw2),
                              P<float>(scratch), heads, S(stream)), "cpb_bwd");
  });
  m.def("cpb_bwd_scratch_floats", [](int heads) { return ddl::cpb_bwd_scratch_floats(heads); });
  m.def("merge_gather", [](ptr_t src, ptr_t dst, int N, int H, int W, int C, bool forward, int sms, ptr_t stream) {
    check(ddl::launch_merge_gather(P<const __nv_bfloat16>(src), P<__nv_bfloat16>(dst), N, H, W, C, forward, sms,
                                   S(stream)), "merge_gather");
  });
  // ------------------------------------------------------------------ squeeze-excitation
  m.def("se_scale", [](ptr_t x, ptr_t s, int lds, ptr_t y, int N, int HW, int C, int sms, ptr_t stream) {
    check(ddl::launch_se_scale(P<const __nv_bfloat16>(x), P<const __nv_bfloat16>(s), lds, P<__nv_bfloat16>(y), N, HW, C,
                               sms, S(stream)), "se_scale");
  });
  m.def("se_reduce", [](ptr_t dy, ptr_t x, ptr_t s, int lds, ptr_t ds, int ldd, int N, int HW, int C, ptr_t stream) {
    check(ddl::launch_se_reduce(P<const __nv_bfloat16>(dy), P<const __nv_bfloat16>(x), P<const __nv_bfloat16>(s), lds,
                                P<__nv_bfloat16>(ds), ldd, N, HW, C, S(stream)), "se_reduce");
  });
  m.def("se_apply", [](ptr_t dy, ptr_t s, int lds, ptr_t dpooled, ptr_t dx, int N, int HW, int C, int sms,
                       ptr_t stream) {
    check(ddl::launch_se_apply(P<const __nv_bfloat16>(dy), P<const __nv_bfloat16>(s), lds, P<const __nv_bfloat16>(dpooled),
                               P<__nv_bfloat16>(dx), N, HW, C, sms, S(stream)), "se_apply");
  });
  // sigmoid gate (EfficientNet): same arguments as the hardsigmoid kernels above
  m.def("se_sig_scale", [](ptr_t x, ptr_t s, int lds, ptr_t y, int N, int HW, int C, int sms, ptr_t stream) {
    check(ddl::launch_se_sig_scale(P<const __nv_bfloat16>(x), P<const __nv_bfloat16>(s), lds, P<__nv_bfloat16>(y), N, HW,
                                   C, sms, S(stream)), "se_sig_scale");
  });
  m.def("se_sig_reduce", [](ptr_t dy, ptr_t x, ptr_t s, int lds, ptr_t ds, int ldd, int N, int HW, int C, ptr_t stream) {
    check(ddl::launch_se_sig_reduce(P<const __nv_bfloat16>(dy), P<const __nv_bfloat16>(x), P<const __nv_bfloat16>(s), lds,
                                    P<__nv_bfloat16>(ds), ldd, N, HW, C, S(stream)), "se_sig_reduce");
  });
  m.def("se_sig_apply", [](ptr_t dy, ptr_t s, int lds, ptr_t dpooled, ptr_t dx, int N, int HW, int C, int sms,
                           ptr_t stream) {
    check(ddl::launch_se_sig_apply(P<const __nv_bfloat16>(dy), P<const __nv_bfloat16>(s), lds,
                                   P<const __nv_bfloat16>(dpooled), P<__nv_bfloat16>(dx), N, HW, C, sms, S(stream)),
          "se_sig_apply");
  });
  // bn_*: (sum, sumsq, gamma, beta, mean, invstd, running_mean, running_var, dgamma, dbeta, gamma_grad, beta_grad,
  // eps, momentum) as pointers (0 = none) and two floats; see ShuffleArgs
  using ShBn = std::tuple<ptr_t, ptr_t, ptr_t, ptr_t, ptr_t, ptr_t, ptr_t, ptr_t, ptr_t, ptr_t, ptr_t, ptr_t, float, float>;
  auto sh_bn = [](const ShBn& t) {
    return ddl::ShuffleBn{P<const float>(std::get<0>(t)), P<const float>(std::get<1>(t)), P<const float>(std::get<2>(t)),
                          P<const float>(std::get<3>(t)), P<float>(std::get<4>(t)), P<float>(std::get<5>(t)),
                          P<float>(std::get<6>(t)), P<float>(std::get<7>(t)), std::get<12>(t), std::get<13>(t),
                          P<float>(std::get<8>(t)), P<float>(std::get<9>(t)), P<float>(std::get<10>(t)),
                          P<float>(std::get<11>(t))};
  };
  m.def("shuffle_fwd", [sh_bn](ptr_t a, ptr_t b, ptr_t s0, ptr_t s1, int M, int half, int ld_ab, int ld_s, int split,
                               int a_bn, int train, const ShBn& bn_a, const ShBn& bn_b, int sms, ptr_t stream) {
    ddl::ShuffleArgs p{};
    p.a = P<const __nv_bfloat16>(a); p.b = P<const __nv_bfloat16>(b); p.s0 = P<__nv_bfloat16>(s0); p.s1 = P<__nv_bfloat16>(s1);
    p.M = M; p.half = half; p.ld_ab = ld_ab; p.ld_s = ld_s; p.split = split; p.a_bn = a_bn; p.train = train;
    p.bn_a = sh_bn(bn_a); p.bn_b = sh_bn(bn_b);
    check(ddl::launch_shuffle_fwd(p, sms, S(stream)), "shuffle_fwd");
  });
  m.def("shuffle_bwd", [sh_bn](ptr_t ds0, ptr_t ds1, ptr_t a, ptr_t b, ptr_t da, ptr_t db, int M, int half, int ld_ab,
                               int ld_s, int split, int a_bn, const ShBn& bn_a, const ShBn& bn_b, int sms, ptr_t stream) {
    ddl::ShuffleArgs p{};
    p.ds0 = P<const __nv_bfloat16>(ds0); p.ds1 = P<const __nv_bfloat16>(ds1); p.a = P<const __nv_bfloat16>(a);
    p.b = P<const __nv_bfloat16>(b); p.da = P<__nv_bfloat16>(da); p.db = P<__nv_bfloat16>(db);
    p.M = M; p.half = half; p.ld_ab = ld_ab; p.ld_s = ld_s; p.split = split; p.a_bn = a_bn; p.train = 1;
    p.bn_a = sh_bn(bn_a); p.bn_b = sh_bn(bn_b);
    check(ddl::launch_shuffle_bwd(p, sms, S(stream)), "shuffle_bwd");
  });
  // GoogLeNet (inception.cu).  segs: per segment 25 integers (x, z, dz, dx, ldx, colx, ldz, colz, lddz, coldz, lddx,
  // coldx, C, sum, sumsq, gamma, beta, mean, invstd, running_mean, running_var, dgamma, dbeta, gamma_grad, beta_grad;
  // pointers 0 = none) and (eps, momentum); see BnSeg
  auto bn_seg = [](const std::vector<std::vector<int64_t>>& segs, const std::vector<std::pair<float, float>>& em, int M) {
    if (segs.empty() || segs.size() > static_cast<size_t>(ddl::kSegMax) || em.size() != segs.size())
      throw std::runtime_error("bn_seg: 1..kSegMax segments");
    ddl::BnSegArgs a{};
    a.n = static_cast<int>(segs.size());
    a.M = M;
    for (int i = 0; i < a.n; ++i) {
      const auto& v = segs[i];
      if (v.size() != 25) throw std::runtime_error("bn_seg: 25 fields per segment");
      ddl::BnSeg& g = a.s[i];
      g.x = P<const __nv_bfloat16>(v[0]); g.z = P<__nv_bfloat16>(v[1]); g.dz = P<const __nv_bfloat16>(v[2]);
      g.dx = P<__nv_bfloat16>(v[3]);
      g.ldx = static_cast<int>(v[4]); g.colx = static_cast<int>(v[5]); g.ldz = static_cast<int>(v[6]);
      g.colz = static_cast<int>(v[7]); g.lddz = static_cast<int>(v[8]); g.coldz = static_cast<int>(v[9]);
      g.lddx = static_cast<int>(v[10]); g.coldx = static_cast<int>(v[11]); g.C = static_cast<int>(v[12]);
      g.sum = P<const float>(v[13]); g.sumsq = P<const float>(v[14]); g.gamma = P<const float>(v[15]);
      g.beta = P<const float>(v[16]); g.mean = P<float>(v[17]); g.invstd = P<float>(v[18]);
      g.running_mean = P<float>(v[19]); g.running_var = P<float>(v[20]); g.dgamma = P<float>(v[21]);
      g.dbeta = P<float>(v[22]); g.gamma_grad = P<float>(v[23]); g.beta_grad = P<float>(v[24]);
      g.eps = em[i].first; g.momentum = em[i].second;
    }
    return a;
  };
  m.def("bn_seg_grid_x", [](int M, int chunks, int sms) { return ddl::bn_seg_grid_x(M, chunks, sms); });
  m.def("bn_seg_fwd", [bn_seg](const std::vector<std::vector<int64_t>>& segs,
                               const std::vector<std::pair<float, float>>& em, int M, int train, int sms, ptr_t stream) {
    check(ddl::launch_bn_seg_fwd(bn_seg(segs, em, M), train != 0, sms, S(stream)), "bn_seg_fwd");
  });
  m.def("bn_seg_bwd", [bn_seg](const std::vector<std::vector<int64_t>>& segs,
                               const std::vector<std::pair<float, float>>& em, int M, ptr_t partial, ptr_t done,
                               int grid_x, ptr_t stream) {
    ddl::BnSegArgs a = bn_seg(segs, em, M);
    a.partial = P<float>(partial);
    a.done = P<unsigned int>(done);
    check(ddl::launch_bn_seg_bwd(a, grid_x, S(stream)), "bn_seg_bwd");
  });
  m.def("adaptive_avgpool_fwd", [](ptr_t x, ptr_t y, int N, int H, int W, int C, int Pq, int Q, int sms, ptr_t stream) {
    check(ddl::launch_adaptive_avgpool_fwd(P<const __nv_bfloat16>(x), P<__nv_bfloat16>(y), N, H, W, C, Pq, Q, sms,
                                           S(stream)), "adaptive_avgpool_fwd");
  });
  m.def("adaptive_avgpool_bwd", [](ptr_t dy, ptr_t dx, int N, int H, int W, int C, int Pq, int Q, int sms, ptr_t stream) {
    check(ddl::launch_adaptive_avgpool_bwd(P<const __nv_bfloat16>(dy), P<__nv_bfloat16>(dx), N, H, W, C, Pq, Q, sms,
                                           S(stream)), "adaptive_avgpool_bwd");
  });
  m.def("transpose_rows", [](ptr_t in, ptr_t out, int N, int A, int B, int sms, ptr_t stream) {
    check(ddl::launch_transpose_rows(P<const __nv_bfloat16>(in), P<__nv_bfloat16>(out), N, A, B, sms, S(stream)),
          "transpose_rows");
  });
  // mats: [(src, dst, rows, k, prows, kp, element bytes)]
  m.def("pad_cols",[](const std::vector<std::tuple<ptr_t, ptr_t, int, int, int, int, int>>& mats, ptr_t stream) {
    if (mats.empty() || mats.size() > static_cast<size_t>(ddl::kPadMax)) throw std::runtime_error("pad_cols: 1..kPadMax matrices");
    ddl::PadBatch b{};
    b.n = static_cast<int>(mats.size());
    for (int i = 0; i < b.n; ++i) {
      const auto& t = mats[i];
      b.m[i] = ddl::PadMatrix{P<const void>(std::get<0>(t)), P<void>(std::get<1>(t)), std::get<2>(t), std::get<3>(t),
                              std::get<4>(t), std::get<5>(t), std::get<6>(t)};
    }
    check(ddl::launch_pad_cols(b, S(stream)), "pad_cols");
  });
  // mats: [(src, dst, rows, k, kp, add)]
  m.def("fold_cols", [](const std::vector<std::tuple<ptr_t, ptr_t, int, int, int, int>>& mats, ptr_t stream) {
    if (mats.empty() || mats.size() > static_cast<size_t>(ddl::kPadMax)) throw std::runtime_error("fold_cols: 1..kPadMax matrices");
    ddl::FoldBatch b{};
    b.n = static_cast<int>(mats.size());
    for (int i = 0; i < b.n; ++i) {
      const auto& t = mats[i];
      b.m[i] = ddl::FoldMatrix{P<const void>(std::get<0>(t)), P<void>(std::get<1>(t)), std::get<2>(t), std::get<3>(t),
                               std::get<4>(t), std::get<5>(t)};
    }
    check(ddl::launch_fold_cols(b, S(stream)), "fold_cols");
  });
  m.def("tanh_rows_fwd", [](ptr_t x, ptr_t y, int64_t n, ptr_t stream) {
    check(ddl::launch_tanh_rows_fwd(P<const __nv_bfloat16>(x), P<__nv_bfloat16>(y), n, S(stream)), "tanh_rows_fwd");
  });
  m.def("tanh_rows_bwd", [](ptr_t dy, ptr_t y, ptr_t dx, int64_t n, ptr_t stream) {
    check(ddl::launch_tanh_rows_bwd(P<const __nv_bfloat16>(dy), P<const __nv_bfloat16>(y), P<__nv_bfloat16>(dx), n,
                                    S(stream)), "tanh_rows_bwd");
  });
  m.def("silu_rows_fwd", [](ptr_t x, int ldx, ptr_t y, int ldy, int N, ptr_t stream) {
    check(ddl::launch_silu_rows_fwd(P<const __nv_bfloat16>(x), ldx, P<__nv_bfloat16>(y), ldy, N, S(stream)),
          "silu_rows_fwd");
  });
  m.def("silu_rows_bwd", [](ptr_t dy, int ldy, ptr_t x, int ldx, ptr_t dx, int c_valid, int N, ptr_t stream) {
    check(ddl::launch_silu_rows_bwd(P<const __nv_bfloat16>(dy), ldy, P<const __nv_bfloat16>(x), ldx, P<__nv_bfloat16>(dx),
                                    c_valid, N, S(stream)), "silu_rows_bwd");
  });
  m.def("stochastic_depth_keep", [](ptr_t keep, int n, float p, uint64_t seed, uint64_t offset, ptr_t stream, ptr_t step) {
    check(ddl::launch_stochastic_depth_keep(P<float>(keep), n, p, seed, offset, P<const int64_t>(step), S(stream)),
          "stochastic_depth_keep");
  });
  m.def("channel_stats", [](ptr_t x, ptr_t sum, ptr_t sumsq, int M, int C, int sms, ptr_t stream) {
    check(ddl::launch_channel_stats(P<const __nv_bfloat16>(x), P<float>(sum), P<float>(sumsq), M, C, sms, S(stream)),
          "channel_stats");
  });

  // ------------------------------------------------------------------ pooling
  m.def("maxpool_fwd", [](ptr_t x, ptr_t y, ptr_t argmax, int N, int H, int W, int C, int Pq, int Q, int k,
                          int stride, int pad, ptr_t stream) {
    check(ddl::launch_maxpool_fwd(P<const __nv_bfloat16>(x), P<__nv_bfloat16>(y), P<uint8_t>(argmax),
                                  pool_args(N, H, W, C, Pq, Q, k, stride, pad), S(stream)), "maxpool_fwd");
  });
  m.def("maxpool_bwd", [](ptr_t dy, ptr_t argmax, ptr_t dx, int N, int H, int W, int C, int Pq, int Q, int k,
                          int stride, int pad, ptr_t stream) {
    check(ddl::launch_maxpool_bwd(P<const __nv_bfloat16>(dy), P<const uint8_t>(argmax), P<__nv_bfloat16>(dx),
                                  pool_args(N, H, W, C, Pq, Q, k, stride, pad), S(stream)), "maxpool_bwd");
  });
  m.def("avgpool_fwd", [](ptr_t x, ptr_t y, int N, int H, int W, int C, int Pq, int Q, int k, int stride, int pad,
                          int count_include_pad, ptr_t stream) {
    check(ddl::launch_avgpool_fwd(P<const __nv_bfloat16>(x), P<__nv_bfloat16>(y),
                                  pool_args(N, H, W, C, Pq, Q, k, stride, pad), count_include_pad, S(stream)),
          "avgpool_fwd");
  });
  m.def("avgpool_bwd", [](ptr_t dy, ptr_t dx, int N, int H, int W, int C, int Pq, int Q, int k, int stride, int pad,
                          int count_include_pad, ptr_t stream) {
    check(ddl::launch_avgpool_bwd(P<const __nv_bfloat16>(dy), P<__nv_bfloat16>(dx),
                                  pool_args(N, H, W, C, Pq, Q, k, stride, pad), count_include_pad, S(stream)),
          "avgpool_bwd");
  });
  m.def("global_avgpool_fwd", [](ptr_t x, ptr_t y, int N, int HW, int C, ptr_t stream) {
    check(ddl::launch_global_avgpool_fwd(P<const __nv_bfloat16>(x), P<__nv_bfloat16>(y), N, HW, C, S(stream)),
          "global_avgpool_fwd");
  });
  m.def("global_avgpool_bwd", [](ptr_t dy, ptr_t dx, int N, int HW, int C, ptr_t stream) {
    check(ddl::launch_global_avgpool_bwd(P<const __nv_bfloat16>(dy), P<__nv_bfloat16>(dx), N, HW, C, S(stream)),
          "global_avgpool_bwd");
  });

  // ------------------------------------------------------------------ loss / data / misc
  m.def("softmax_xent", [](ptr_t logits, ptr_t labels, ptr_t dlogits, ptr_t loss_sum, ptr_t per_sample,
                           ptr_t correct, float loss_scale, float grad_scale, int B, int classes, int ld,
                           ptr_t stream) {
    XentArgs a;
    a.logits = P<const __nv_bfloat16>(logits); a.labels = P<const int64_t>(labels);
    a.dlogits = P<__nv_bfloat16>(dlogits); a.loss_sum = P<float>(loss_sum); a.per_sample = P<float>(per_sample);
    a.correct = P<int32_t>(correct); a.loss_scale = loss_scale; a.grad_scale = grad_scale; a.B = B;
    a.classes = classes; a.ld = ld;
    check(ddl::launch_softmax_xent(a, S(stream)), "softmax_xent");
  });
  m.def("philox_normal_nhwc", [](ptr_t out, int64_t pixels, int c_valid, int cpad, uint64_t seed, uint64_t offset,
                                 ptr_t stream) {
    check(ddl::launch_philox_normal_nhwc(P<__nv_bfloat16>(out), pixels, c_valid, cpad, seed, offset, S(stream)),
          "philox_normal_nhwc");
  });
  m.def("philox_labels", [](ptr_t out, int64_t n, int classes, uint64_t seed, uint64_t offset, ptr_t stream) {
    check(ddl::launch_philox_labels(P<int64_t>(out), n, classes, seed, offset, S(stream)), "philox_labels");
  });
  m.def("nchw_to_nhwc_norm", [](ptr_t in, ptr_t out, int N, int C, int H, int W, int cpad, ptr_t mean, ptr_t stdv,
                                ptr_t stream) {
    check(ddl::launch_nchw_to_nhwc_norm(P<const float>(in), P<__nv_bfloat16>(out), N, C, H, W, cpad,
                                        P<const float>(mean), P<const float>(stdv), S(stream)), "nchw_to_nhwc_norm");
  });
  m.def("nhwc_u8_to_nhwc4", [](ptr_t in, ptr_t out, int64_t pixels, ptr_t mean, ptr_t stdv, ptr_t stream) {
    check(ddl::launch_nhwc_u8_to_nhwc4(P<const uint8_t>(in), P<__nv_bfloat16>(out), pixels, P<const float>(mean),
                                       P<const float>(stdv), S(stream)), "nhwc_u8_to_nhwc4");
  });
  // ------------------------------------------------------------------ fp8 operand preparation
  m.attr("FP8_SLOT_BYTES") = static_cast<int>(sizeof(ddl::Fp8Slot));
  m.def("fp8_quantize", [](ptr_t x, ptr_t out, int64_t n, ptr_t slot, bool e5m2, int sms, ptr_t stream) {
    check(ddl::launch_fp8_quantize(P<const __nv_bfloat16>(x), P<uint8_t>(out), n, P<ddl::Fp8Slot>(slot), e5m2, sms,
                                   S(stream)), "fp8_quantize");
  });
  m.def("fp8_quantize_mx", [](ptr_t x, ptr_t out, ptr_t sf, int64_t rows, int64_t K, int sms, ptr_t stream) {
    check(ddl::launch_fp8_quantize_mx(P<const __nv_bfloat16>(x), P<uint8_t>(out), P<uint8_t>(sf), rows, K, sms, S(stream)),
          "fp8_quantize_mx");
  }, "bf16 [rows][K] -> e4m3 [rows][K] + UE8M0 block scales (32 elements) in the tensor core's 512-byte atom order");
  m.def("fp8_amax", [](ptr_t x, int64_t n, ptr_t slot, int sms, ptr_t stream) {
    check(ddl::launch_fp8_amax(P<const __nv_bfloat16>(x), n, P<ddl::Fp8Slot>(slot), sms, S(stream)), "fp8_amax");
  });
  m.def("fp8_transpose_taps", [](ptr_t in, ptr_t out, int rows, int taps, int cols, ptr_t stream) {
    check(ddl::launch_fp8_transpose_taps(P<const uint8_t>(in), P<uint8_t>(out), rows, taps, cols, S(stream)),
          "fp8_transpose_taps");
  });
  m.def("fp8_update_scales", [](ptr_t slots, int n, ptr_t stream) {
    check(ddl::launch_fp8_update_scales(P<ddl::Fp8Slot>(slots), n, S(stream)), "fp8_update_scales");
  });
  m.def("cast_f32_bf16", [](ptr_t in, ptr_t out, int64_t n, ptr_t stream) {
    check(ddl::launch_cast_f32_bf16(P<const float>(in), P<__nv_bfloat16>(out), n, S(stream)), "cast_f32_bf16");
  });
  m.def("pack_stem_weight", [](ptr_t w, ptr_t packed, int Cout, int R, int Sx, int Cin, int RP, int SP,
                               ptr_t stream) {
    check(ddl::launch_pack_stem_weight(P<const float>(w), P<__nv_bfloat16>(packed), Cout, R, Sx, Cin, RP, SP,
                                       S(stream)), "pack_stem_weight");
  });
  m.def("unpack_stem_grad", [](ptr_t packed, ptr_t gw, int Cout, int R, int Sx, int Cin, int RP, int SP,
                               ptr_t stream) {
    check(ddl::launch_unpack_stem_grad(P<const float>(packed), P<float>(gw), Cout, R, Sx, Cin, RP, SP, S(stream)),
          "unpack_stem_grad");
  });
  m.def("bias_relu_bwd", [](ptr_t dy, ptr_t z, ptr_t dx, ptr_t dbias, int M, int C, int c_valid, int relu, int sms,
                            ptr_t stream) {
    check(ddl::launch_bias_relu_bwd(P<const __nv_bfloat16>(dy), P<const __nv_bfloat16>(z), P<__nv_bfloat16>(dx),
                                    P<float>(dbias), M, C, c_valid, relu, sms, S(stream)), "bias_relu_bwd");
  });
  m.def("dropout", [](ptr_t x, ptr_t y, int64_t n, float p, uint64_t seed, uint64_t offset, ptr_t stream, ptr_t step) {
    check(ddl::launch_dropout(P<const __nv_bfloat16>(x), P<__nv_bfloat16>(y), n, p, seed, offset, P<const int64_t>(step),
                              S(stream)), "dropout");
  }, py::arg("x"), py::arg("y"), py::arg("n"), py::arg("p"), py::arg("seed"), py::arg("offset"), py::arg("stream"),
     py::arg("step") = 0);
  m.def("pad_nhwc4", [](ptr_t in, ptr_t out, int N, int H, int W, int Hp, int Wp, int pt, int pl, int G, ptr_t stream) {
    check(ddl::launch_pad_nhwc4(P<const __nv_bfloat16>(in), P<__nv_bfloat16>(out), N, H, W, Hp, Wp, pt, pl, G, S(stream)),
          "pad_nhwc4");
  });
  m.def("concat_channels", [](std::vector<ptr_t> parts, std::vector<int> chans, ptr_t whole, int M, bool scatter,
                              ptr_t stream) {
    ddl::CatArgs a;
    if (parts.size() != chans.size() || parts.empty() || parts.size() > static_cast<size_t>(ddl::kCatMax))
      throw std::runtime_error("concat_channels: 1..8 parts");
    a.n = static_cast<int>(parts.size());
    a.ctot = 0;
    for (int i = 0; i < ddl::kCatMax; ++i) {
      a.part[i] = i < a.n ? P<__nv_bfloat16>(parts[i]) : nullptr;
      a.c[i] = i < a.n ? chans[i] : 0;
      a.ctot += a.c[i];
    }
    a.whole = P<__nv_bfloat16>(whole); a.M = M;
    check(ddl::launch_concat_channels(a, scatter, S(stream)), "concat_channels");
  });
  m.def("hardswish_fwd", [](ptr_t x, ptr_t y, int64_t n, ptr_t stream) {
    check(ddl::launch_hardswish_fwd(P<const __nv_bfloat16>(x), P<__nv_bfloat16>(y), n, S(stream)), "hardswish_fwd");
  });
  m.def("hardswish_bwd", [](ptr_t dy, ptr_t x, ptr_t dx, int64_t n, ptr_t stream) {
    check(ddl::launch_hardswish_bwd(P<const __nv_bfloat16>(dy), P<const __nv_bfloat16>(x), P<__nv_bfloat16>(dx), n,
                                    S(stream)), "hardswish_bwd");
  });
  m.def("add_bf16", [](ptr_t a, ptr_t b, ptr_t y, int64_t n, ptr_t stream) {
    check(ddl::launch_add_bf16(P<const __nv_bfloat16>(a), P<const __nv_bfloat16>(b), P<__nv_bfloat16>(y), n,
                               S(stream)), "add_bf16");
  });
}
