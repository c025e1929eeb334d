// Python bindings of the sm_90a kernels.  Ops are thin objects that own a filled launch
// struct (raw device addresses supplied by Python, which keeps the tensors alive) and launch on
// PyTorch's current CUDA stream, so they compose with torch.cuda.graph capture: a whole
// consensus round is captured once and replayed.
#include <torch/extension.h>
#include <cstring>
#include <string>
#include <ATen/cuda/CUDAContext.h>
#include <pybind11/pybind11.h>

#include "consensus.h"
#include "mnist.h"

namespace py = pybind11;
using namespace nndt;

static inline cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }
static inline void check(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}
template <typename P> static P* ptr(const py::dict& d, const char* k) {
  if (!d.contains(k) || d[k].is_none()) return nullptr;
  return reinterpret_cast<P*>(d[k].cast<uint64_t>());
}
static int geti(const py::dict& d, const char* k, int dflt = 0) { return d.contains(k) ? d[k].cast<int>() : dflt; }
static double getf(const py::dict& d, const char* k, double dflt = 0) { return d.contains(k) ? d[k].cast<double>() : dflt; }

// ------------------------------------------------------------------ MNIST ----
struct MnistOp {
  mnist::Args a{};
  mnist::GenericShape gs{3, 5, 64, 0, 0.0, 1.0};
  int spb = 8, S = 1, eval_ctas = 1, generic = 0, tc = 0, cl64 = 0;
  alignas(64) unsigned char w1_map[128] = {0};
  explicit MnistOp(const py::dict& d) { update(d); }
  void update(const py::dict& d) {
    a.theta = ptr<const float>(d, "theta"); a.n_pad = geti(d, "n_pad"); a.L = geti(d, "L");
    a.off_wc = geti(d, "off_wc"); a.off_bc = geti(d, "off_bc"); a.off_w1 = geti(d, "off_w1");
    a.off_b1 = geti(d, "off_b1"); a.off_w2 = geti(d, "off_w2"); a.off_b2 = geti(d, "off_b2");
    a.x = ptr<const void>(d, "x"); a.y = ptr<const int64_t>(d, "y");
    a.x_is_u8 = geti(d, "x_is_u8"); a.mean = (float)getf(d, "mean"); a.inv_std = (float)getf(d, "inv_std", 1.0);
    a.direct = geti(d, "direct"); a.batch = geti(d, "batch"); a.seed = geti(d, "seed"); a.node0 = geti(d, "node0");
    a.shard_off = ptr<const int>(d, "shard_off"); a.shard_len = ptr<const int>(d, "shard_len");
    a.calls = ptr<int>(d, "calls"); a.arrive = ptr<unsigned int>(d, "arrive"); a.tune = geti(d, "tune", 1); a.prof = ptr<long long>(d, "step_prof"); a.direct_bs = ptr<const int>(d, "direct_bs");
    a.grad_part = ptr<float>(d, "grad_part"); a.loss_part = ptr<float>(d, "loss_part"); a.loss_mirror = ptr<float>(d, "loss_mirror");
    a.n_val = geti(d, "n_val"); a.val_loss = ptr<float>(d, "val_loss");
    a.val_correct = ptr<unsigned char>(d, "val_correct");
    spb = geti(d, "spb", 8); S = geti(d, "S", 1); eval_ctas = geti(d, "eval_ctas", 1);
    // generic CUDA-core kernel (mnist_generic.cu): any conv shape, fp32 / fp64 (theta, grad_part, val_loss then address doubles)
    generic = geti(d, "generic", 0);
    gs.F = geti(d, "num_filters", 3); gs.KS = geti(d, "kernel_size", 5); gs.LW = geti(d, "linear_width", 64);
    gs.dtype64 = geti(d, "dtype64", 0); gs.mean = getf(d, "mean"); gs.inv_std = getf(d, "inv_std", 1.0);
    // K-split cluster kernel (mnist_tc.cu): needs the W1 tensor map
    cl64 = geti(d, "cl64", 0);
    tc = geti(d, "tc", 0);
    if (tc) {
      const std::string m = d["w1_map"].cast<py::bytes>();
      if (m.size() != 128) throw std::runtime_error("w1_map must be the 128-byte CUtensorMap");
      memcpy(w1_map, m.data(), 128);
    }
  }
  void train() {
    if (cl64) check(mnist::launch_train_cl64(a, gs, S, cur_stream()), "mnist_cl64_train");
    else if (generic) check(mnist::launch_generic_train(a, gs, spb, S, cur_stream()), "convnet_generic_train");
    else if (tc) check(mnist::launch_train_tc(a, w1_map, S, cur_stream()), "mnist_tc_train");
    else check(mnist::launch_train(a, spb, S, cur_stream()), "mnist_train");
  }
  void eval() {
    if (generic) check(mnist::launch_generic_eval(a, gs, eval_ctas, cur_stream()), "convnet_generic_eval");
    else check(mnist::launch_eval(a, eval_ctas, cur_stream()), "mnist_eval");
  }
};

struct GatherOp {
  mnist::GatherArgs a{};
  explicit GatherOp(const py::dict& d) {
    a.x_host = ptr<const unsigned char>(d, "x_host"); a.y_host = ptr<const int64_t>(d, "y_host");
    a.row_bytes = geti(d, "row_bytes"); a.x_stage = ptr<unsigned char>(d, "x_stage");
    a.y_stage = ptr<int64_t>(d, "y_stage"); a.bs_stage = ptr<int>(d, "bs_stage");
    a.P = geti(d, "P"); a.L = geti(d, "L"); a.batch = geti(d, "batch"); a.seed = geti(d, "seed"); a.node0 = geti(d, "node0");
    a.shard_off = ptr<const int>(d, "shard_off"); a.shard_len = ptr<const int>(d, "shard_len");
    a.calls0 = ptr<const int>(d, "calls0"); a.stage_round = ptr<int>(d, "stage_round");
    a.done_ctr = ptr<unsigned int>(d, "done_ctr"); a.max_blocks = geti(d, "max_blocks", 24);
  }
  void launch() { check(mnist::launch_gather(a, cur_stream()), "gather_rows"); }
};

// -------------------------------------------------------------- consensus ----
template <typename T>
static consensus::Common<T> common_from(const py::dict& d) {
  consensus::Common<T> c{};
  c.L = geti(d, "L"); c.n_pad = geti(d, "n_pad"); c.S = geti(d, "S", 1);
  c.theta = ptr<T>(d, "theta"); c.grad_part = ptr<const T>(d, "grad_part");
  c.pub = ptr<T>(d, "pub"); c.C = geti(d, "C", 1); c.pub_L = geti(d, "pub_L", c.L);
  c.nbr_ptr = ptr<const int64_t>(d, "nbr_ptr"); c.nbr_w = ptr<const T>(d, "nbr_w");
  c.self_w = ptr<const T>(d, "self_w"); c.deg = ptr<const int>(d, "deg");
  c.nbr_rank = ptr<const int>(d, "nbr_rank"); c.dmax = geti(d, "dmax");
  c.rdr_deg = ptr<const int>(d, "rdr_deg"); c.rdr_rank = ptr<const int>(d, "rdr_rank"); c.rmax = geti(d, "rmax", 1);
  c.round_ctr = ptr<int>(d, "round_ctr");
  c.rho = ptr<const T>(d, "rho"); c.lr = ptr<const T>(d, "lr"); c.alpha = ptr<const T>(d, "alpha");
  c.graph_id = ptr<const int>(d, "graph_id");
  c.calls = ptr<int>(d, "calls");
  c.loss_part = ptr<const float>(d, "loss_part"); c.tloss = ptr<float>(d, "tloss");
  c.tdecay = (float)getf(d, "tdecay", 0.0); c.loss_S = geti(d, "loss_S", 1);
  c.flags = ptr<int>(d, "flags"); c.peer_flag = ptr<const int64_t>(d, "peer_flag");
  c.world = geti(d, "world", 1); c.rank = geti(d, "rank", 0);
  c.done_ctr = ptr<unsigned int>(d, "done_ctr"); c.err = ptr<int>(d, "err");
  c.notify_mask = d.contains("notify_mask") ? d["notify_mask"].cast<unsigned long long>() : ~0ull;
  c.node_order = ptr<const int>(d, "node_order");
  c.timeline = ptr<long long>(d, "timeline");
  c.pub_seq = ptr<int>(d, "pub_seq"); c.nbr_seq = ptr<const int64_t>(d, "nbr_seq");
  c.sum_mode = geti(d, "sum_mode", 0); c.n_total = geti(d, "n_total", 0);
  c.sum_local = ptr<double>(d, "sum_local"); c.sum_mc = ptr<const double>(d, "sum_mc");
  c.sum_flags = ptr<int>(d, "sum_flags"); c.peer_sum_flag = ptr<const int64_t>(d, "peer_sum_flag");
  return c;
}

template <typename T>
struct ConsensusOp {
  consensus::Common<T> c{};
  consensus::DinnoArgs<T> dn{};
  consensus::DsgtArgs<T> gt{};
  consensus::EdArgs<T> ed{};
  consensus::MomentumArgs<T> mo{};
  bool mo_qg = false;
  consensus::ChocoArgs<T> ch{};
  consensus::BeerArgs<T> be{};
  consensus::KgtArgs<T> kg{};
  consensus::DetagArgs<T> dt{};
  consensus::HsgdArgs<T> hs{};
  consensus::XgArgs<T> xg{};
  consensus::PgaArgs<T> pa{};
  consensus::SlowmoArgs<T> sm{};
  consensus::DpArgs<T> dp{};
  consensus::MoniquaArgs<T> mq{};
  consensus::SparqArgs<T> sq{};
  consensus::DAdaptiveArgs<T> ad{};
  consensus::RelayArgs<T> rs{};
  consensus::PgArgs<T> pg{};
  consensus::ClipArgs<T> cg{};
  int cg_adaptive = 0;
  consensus::ScreenArgs<T> br{};
  consensus::SgpArgs<T> sg{};
  consensus::PushDigArgs<T> pd{};
  explicit ConsensusOp(const py::dict& d) {
    c = common_from<T>(d);
    dn.c = c; gt.c = c; ed.c = c; mo.c = c; ch.c = c; be.c = c; kg.c = c; ad.c = c; rs.c = c; cg.c = c; br.c = c; sg.c = c;
    pd.c = c; pg.c = c; dt.c = c; hs.c = c; pa.c = c; dp.c = c; mq.c = c; sq.c = c; xg.c = c; sm.c = c;
    xg.xmix = ptr<T>(d, "xmix"); xg.theta_x = ptr<T>(d, "theta_x"); xg.grad_part_x = ptr<const T>(d, "grad_part_x");
    xg.g = ptr<T>(d, "xg_g"); xg.coef0 = ptr<const double>(d, "xg_coef0"); xg.coef = ptr<const double>(d, "xg_coef");
    pg.vec = ptr<T>(d, "pg_vec"); pg.seg = ptr<const int>(d, "pg_seg"); pg.sign = ptr<const int>(d, "pg_sign");
    pg.nseg = geti(d, "pg_nseg", 0); pg.P = geti(d, "pg_P", 0); pg.Q = geti(d, "pg_Q", 0); pg.B = geti(d, "pg_B", 0);
    pg.W = geti(d, "pg_W", 0); pg.gamma = (T)getf(d, "gamma", 1.0); pg.grid_x = geti(d, "pg_grid", 0);
    br.b = geti(d, "screen_b", -1); br.median = geti(d, "screen_median", 0);
    sg.x = ptr<T>(d, "x"); sg.w = ptr<double>(d, "w");
    sg.row_stride = d.contains("row_stride") ? d["row_stride"].cast<long long>() : 0;
    pd.u = ptr<T>(d, "u"); pd.w = sg.w; pd.ysum = ptr<T>(d, "ysum"); pd.g_old = ptr<T>(d, "g_old");
    pd.row_stride = sg.row_stride;
    ed.psi = ptr<T>(d, "psi");
    mo_qg = geti(d, "quasi_global", 0) != 0;
    mo.m = ptr<T>(d, "m"); mo.x_prev = mo_qg ? ptr<T>(d, "x_prev") : nullptr;
    mo.beta = (T)getf(d, "beta", 0.0); mo.nesterov = geti(d, "nesterov", 0);
    ch.x_hat = ptr<T>(d, "x_hat"); ch.s = ptr<T>(d, "s"); ch.live = ptr<const unsigned>(d, "live");
    ch.gamma = (T)getf(d, "gamma", 1.0); ch.code = geti(d, "code", 0);
    ch.code_stride = d.contains("code_stride") ? d["code_stride"].cast<long long>() : 0;
    ch.topk_k = geti(d, "topk_k", 0);
    be.h = ptr<T>(d, "h"); be.s_h = ptr<T>(d, "s_h"); be.v = ptr<T>(d, "v"); be.g = ptr<T>(d, "g");
    be.s_g = ptr<T>(d, "s_g"); be.m_old = ptr<T>(d, "m_old");
    be.live = ch.live; be.gamma = ch.gamma; be.code = ch.code; be.code_stride = ch.code_stride; be.topk_k = ch.topk_k;
    kg.corr = ptr<T>(d, "corr"); kg.dacc = ptr<T>(d, "dacc");
    kg.K = geti(d, "local_steps", 1); kg.correction = geti(d, "correction", 1);
    dt.omega = ptr<const T>(d, "omega"); dt.ymix = ptr<T>(d, "ymix"); dt.g_old = ptr<T>(d, "g_old");
    dt.K = geti(d, "gossip_steps", 0);
    hs.grad_part_prev = ptr<const T>(d, "grad_part_prev"); hs.v = ptr<T>(d, "hsgd_v"); hs.theta_prev = ptr<T>(d, "theta_prev");
    hs.omb = (T)getf(d, "omb", 0.0);
    pa.period = geti(d, "period", 0); pa.gossip = geti(d, "gossip", 1);
    sm.anchor = ptr<T>(d, "anchor"); sm.u = ptr<T>(d, "slow_u"); sm.m = ptr<T>(d, "m"); sm.period = pa.period;
    sm.alpha0 = (T)getf(d, "alpha0", 0.0); sm.slow_lr = getf(d, "slow_lr", 1.0);
    sm.slow_momentum = getf(d, "slow_momentum", 0.0);
    dp.norm_part = ptr<double>(d, "norm_part"); dp.pstride = geti(d, "pstride", 0);
    dp.nbr_id = ptr<const int>(d, "nbr_id"); dp.live = ptr<const unsigned>(d, "live"); dp.node0 = geti(d, "node0", 0);
    dp.clip = getf(d, "clip_norm", 0.0); dp.cz_dp = getf(d, "cz_dp", 0.0); dp.cz_pair = getf(d, "cz_pair", 0.0);
    dp.key0 = d.contains("dp_key0") ? (unsigned)d["dp_key0"].cast<unsigned long long>() : 0u;
    dp.key1 = d.contains("dp_key1") ? (unsigned)d["dp_key1"].cast<unsigned long long>() : 0u;
    mq.psi = ptr<T>(d, "psi"); mq.live = ptr<const unsigned>(d, "live"); mq.B = getf(d, "mq_B", 0.0);
    mq.bits = geti(d, "mq_bits", 0); mq.node0 = geti(d, "node0", 0); mq.margin = ptr<unsigned long long>(d, "mq_margin");
    mq.key0 = d.contains("mq_key0") ? (unsigned)d["mq_key0"].cast<unsigned long long>() : 0u;
    mq.key1 = d.contains("mq_key1") ? (unsigned)d["mq_key1"].cast<unsigned long long>() : 0u;
    mq.code_stride = d.contains("code_stride") ? d["code_stride"].cast<long long>() : 0;
    sq.x_hat = ptr<T>(d, "x_hat"); sq.s = ptr<T>(d, "s"); sq.live = ptr<const unsigned>(d, "live");
    sq.thr = ptr<const double>(d, "sparq_thr"); sq.norm_part = ptr<double>(d, "norm_part"); sq.pstride = geti(d, "pstride", 0);
    sq.triggers = ptr<long long>(d, "sparq_triggers"); sq.gamma = (T)getf(d, "gamma", 1.0); sq.code = geti(d, "code", 0);
    sq.code_bytes = d.contains("sparq_code_bytes") ? d["sparq_code_bytes"].cast<long long>() : 0;
    sq.row_stride = d.contains("row_stride") ? d["row_stride"].cast<long long>() : 0;
    sq.H = geti(d, "local_steps", 1);
    ad.m = ptr<T>(d, "ad_m"); ad.v = ptr<T>(d, "ad_v"); ad.vhat = ptr<T>(d, "vhat"); ad.ut = ptr<T>(d, "ut");
    ad.beta1 = (T)getf(d, "beta1", 0.9); ad.beta2 = (T)getf(d, "beta2", 0.999); ad.eps = (T)getf(d, "ad_eps", 1e-8);
    ad.adagrad = geti(d, "adagrad", 0); ad.tracking = geti(d, "tracking", 1);
    rs.reach = ptr<const T>(d, "reach"); rs.rin = ptr<T>(d, "rin"); rs.diam = geti(d, "diam", 0);
    rs.n = (T)geti(d, "relay_n", 0);
    cg.dist_part = ptr<double>(d, "dist_part"); cg.pstride = geti(d, "pstride", 0);
    cg.attack = ptr<const int>(d, "attack"); cg.nbr_byz = ptr<const int>(d, "nbr_byz");
    cg.delta = getf(d, "clip_delta", 0.0); cg.scale = getf(d, "attack_scale", 1.0); cg.z = getf(d, "attack_z", 1.0);
    cg_adaptive = geti(d, "clip_adaptive", 0);
    dn.dual = ptr<T>(d, "dual"); dn.delta = ptr<T>(d, "delta"); dn.m = ptr<T>(d, "m"); dn.v = ptr<T>(d, "v");
    dn.pits = geti(d, "pits", 1); dn.opt = geti(d, "opt", 1); dn.persistent = geti(d, "persistent", 0);
    gt.g_old = ptr<T>(d, "g_old");
    gt.alpha_row = ptr<const T>(d, "alpha_row"); gt.own_tracker = geti(d, "own_tracker", 0);
  }
  void dinno_update(int step) {
    dn.step = step;
    check(consensus::launch_dinno_update<T>(dn, cur_stream()), "dinno_update");
  }
  void local_sum() { check(consensus::launch_local_sum<T>(c, cur_stream()), "local_sum"); }
  void dsgd_mix() { check(consensus::launch_dsgd_mix<T>(c, cur_stream()), "dsgd_mix"); }
  void dsgd_step() { check(consensus::launch_dsgd_step<T>(c, cur_stream()), "dsgd_step"); }
  void dsgt_init() { check(consensus::launch_dsgt_init<T>(gt, cur_stream()), "dsgt_init"); }
  void dsgt_mix() { check(consensus::launch_dsgt_mix<T>(gt, cur_stream()), "dsgt_mix"); }
  void dsgt_track() { check(consensus::launch_dsgt_track<T>(gt, cur_stream()), "dsgt_track"); }
  void ed_mix() { check(consensus::launch_ed_mix<T>(ed, cur_stream()), "ed_mix"); }
  void ed_step() {
    if (ed.psi == nullptr) throw std::runtime_error("ed_step needs the Exact Diffusion row `psi`");
    check(consensus::launch_ed_step<T>(ed, cur_stream()), "ed_step");
  }
  void dsgdm_step() {
    if (mo.m == nullptr || (mo_qg && mo.x_prev == nullptr))
      throw std::runtime_error("dsgdm_step needs the momentum row `m` (and `x_prev` with quasi-global momentum)");
    check(consensus::launch_dsgdm_step<T>(mo, cur_stream()), "dsgdm_step");
  }
  void choco_check(const char* what) const {
    if (ch.x_hat == nullptr || ch.s == nullptr || ch.live == nullptr || ch.code_stride <= 0)
      throw std::runtime_error(std::string(what) + " needs the CHOCO rows `x_hat`, `s`, the `live` mask and `code_stride`");
  }
  void choco_mix() {
    choco_check("choco_mix");
    check(consensus::launch_choco_mix<T>(ch, cur_stream()), "choco_mix");
  }
  void choco_step() {
    choco_check("choco_step");
    check(consensus::launch_choco_step<T>(ch, cur_stream()), "choco_step");
  }
  void beer_check(const char* what) const {
    if (be.h == nullptr || be.s_h == nullptr || be.v == nullptr || be.g == nullptr || be.s_g == nullptr ||
        be.m_old == nullptr || be.live == nullptr || be.code_stride <= 0 || c.C != 2)
      throw std::runtime_error(std::string(what) + " needs the BEER rows `h`, `s_h`, `v`, `g`, `s_g`, `m_old`, the `live` "
                               "mask, `code_stride` and two published channels");
  }
  void beer_mix() {
    beer_check("beer_mix");
    check(consensus::launch_beer_mix<T>(be, cur_stream()), "beer_mix");
  }
  void beer_step() {
    beer_check("beer_step");
    check(consensus::launch_beer_step<T>(be, cur_stream()), "beer_step");
  }
  void kgt_mix() {
    if (!kg.correction || kg.corr == nullptr || c.C != 2)
      throw std::runtime_error("kgt_mix needs correction mode, the K-GT row `corr` and two published channels "
                               "(local DSGD mixes with dsgd_mix)");
    check(consensus::launch_kgt_mix<T>(kg, cur_stream()), "kgt_mix");
  }
  void kgt_step(int step) {
    if (kg.K < 1 || step < 0 || step >= kg.K)
      throw std::runtime_error("kgt_step: step " + std::to_string(step) + " outside 0.." + std::to_string(kg.K - 1));
    if (kg.correction && (kg.corr == nullptr || kg.dacc == nullptr || c.C != 2))
      throw std::runtime_error("kgt_step with correction needs the K-GT rows `corr`, `dacc` and two published channels");
    kg.step = step;
    check(consensus::launch_kgt_step<T>(kg, cur_stream()), "kgt_step");
  }
  void detag_check(const char* what) const {
    if (dt.omega == nullptr || dt.ymix == nullptr || dt.g_old == nullptr || dt.K < 1 || c.sum_mode || c.C != 2)
      throw std::runtime_error(std::string(what) + " needs the sub-step weights `omega`, the rows `ymix` and `g_old`, "
                               "`gossip_steps` >= 1, the pointer-table neighbors and two published channels");
  }
  void ag_gossip(int step) {
    detag_check("ag_gossip");
    if (step < 0 || step >= dt.K)
      throw std::runtime_error("ag_gossip: sub-step " + std::to_string(step) + " outside 0.." + std::to_string(dt.K - 1));
    dt.step = step;
    check(consensus::launch_ag_gossip<T>(dt, cur_stream()), "ag_gossip");
  }
  void detag_track() {
    detag_check("detag_track");
    check(consensus::launch_detag_track<T>(dt, cur_stream()), "detag_track");
  }
  void hsgd_track() {
    if (hs.grad_part_prev == nullptr || hs.v == nullptr || hs.theta_prev == nullptr || c.C != 2)
      throw std::runtime_error("hsgd_track needs the prev-point partials `grad_part_prev`, the rows `hsgd_v` and "
                               "`theta_prev` and two published channels");
    check(consensus::launch_hsgd_track<T>(hs, cur_stream()), "hsgd_track");
  }
  void pga_check(const char* what) const {
    if (pa.period < 1 || c.sum_local == nullptr || c.sum_mode || c.C != 1 || c.n_total < 1)
      throw std::runtime_error(std::string(what) + " needs `period` >= 1, the fp64 partial-sum buffer `sum_local`, "
                               "`n_total`, the pointer-table neighbors and one published channel");
  }
  void pga_sum() {
    pga_check("pga_sum");
    check(consensus::launch_pga_sum<T>(pa, cur_stream()), "pga_sum");
  }
  void pga_mix() {
    pga_check("pga_mix");
    check(consensus::launch_pga_mix<T>(pa, cur_stream()), "pga_mix");
  }
  void slowmo_outer() {
    if (sm.period < 1 || sm.anchor == nullptr || sm.u == nullptr || c.C != 1)
      throw std::runtime_error("slowmo_outer needs `period` >= 1, the SlowMo rows `anchor` and `slow_u` and one "
                               "published channel");
    check(consensus::launch_slowmo_outer<T>(sm, cur_stream()), "slowmo_outer");
  }
  void dp_check(const char* what) const {
    if (dp.norm_part == nullptr || dp.pstride <= 0 || dp.nbr_id == nullptr || dp.live == nullptr || !(dp.clip > 0.0) ||
        c.C != 1 || c.sum_mode)
      throw std::runtime_error(std::string(what) + " needs the fp64 norm partials `norm_part` and `pstride`, the "
                               "neighbor id table `nbr_id`, the `live` mask, `clip_norm` > 0, one published channel and "
                               "the pointer-table neighbors");
  }
  void dp_norm() {
    dp_check("dp_norm");
    check(consensus::launch_dp_norm<T>(dp, cur_stream()), "dp_norm");
  }
  void dp_step() {
    dp_check("dp_step");
    check(consensus::launch_dp_step<T>(dp, cur_stream()), "dp_step");
  }
  void mq_check(const char* what) const {
    if (!(mq.bits == 2 || mq.bits == 4 || mq.bits == 8) || mq.live == nullptr || mq.margin == nullptr || !(mq.B > 0.0) ||
        c.n_pad % 128 != 0 || mq.code_stride != (long long)c.n_pad * mq.bits / 8 || c.C != 1 || c.sum_mode)
      throw std::runtime_error(std::string(what) + " needs `mq_bits` in {2, 4, 8}, the `live` mask, the `mq_margin` "
                               "counters, `mq_B` > 0, rows padded to a multiple of 128, `code_stride` = n_pad * bits / 8, "
                               "one published channel and the pointer-table neighbors");
  }
  void sparq_check(const char* what) const {
    if (sq.x_hat == nullptr || sq.s == nullptr || sq.live == nullptr || sq.thr == nullptr || sq.norm_part == nullptr ||
        sq.triggers == nullptr || sq.pstride <= 0 || sq.H < 1 || sq.code_bytes <= 0 || sq.code_bytes % 16 != 0 ||
        sq.row_stride != sq.code_bytes + 16 || c.n_pad % 128 != 0 || c.dmax > 256 || c.C != 1 || c.sum_mode ||
        !(sq.code == 0 || sq.code == 1 || sq.code == 2))
      throw std::runtime_error(std::string(what) + " needs the SPARQ rows `x_hat`, `s`, the `live` mask, the threshold "
                               "schedule `sparq_thr`, the fp64 partials `norm_part` and `pstride`, the `sparq_triggers` "
                               "counters, `local_steps` >= 1, a code of none / int8 / sign with `sparq_code_bytes` (a "
                               "multiple of 16) and `row_stride` = sparq_code_bytes + 16, rows padded to a multiple of "
                               "128, at most 256 neighbors, one published channel and the pointer-table neighbors");
  }
  void sparq_mix() {
    sparq_check("sparq_mix");
    check(consensus::launch_sparq_mix<T>(sq, cur_stream()), "sparq_mix");
  }
  void sparq_step(int step) {
    sparq_check("sparq_step");
    if (step < 0 || step >= sq.H)
      throw std::runtime_error("sparq_step: step " + std::to_string(step) + " outside 0.." + std::to_string(sq.H - 1));
    sq.step = step;
    check(consensus::launch_sparq_step<T>(sq, cur_stream()), "sparq_step");
  }
  void sparq_publish() {
    sparq_check("sparq_publish");
    check(consensus::launch_sparq_publish<T>(sq, cur_stream()), "sparq_publish");
  }
  void mq_mix() {
    mq_check("mq_mix");
    check(consensus::launch_mq_mix<T>(mq, cur_stream()), "mq_mix");
  }
  void mq_step() {
    mq_check("mq_step");
    check(consensus::launch_mq_step<T>(mq, cur_stream()), "mq_step");
  }
  void dadaptive_mix() {
    if (!ad.tracking || ad.ut == nullptr || c.C != 2)
      throw std::runtime_error("dadaptive_mix needs tracking, the tracker row `ut` and two published channels (the "
                               "own-second-moment variant mixes with dsgd_mix)");
    check(consensus::launch_dadaptive_mix<T>(ad, cur_stream()), "dadaptive_mix");
  }
  void dadaptive_step() {
    if (ad.m == nullptr || ad.vhat == nullptr || (!ad.adagrad && ad.v == nullptr) ||
        (ad.tracking && (ad.ut == nullptr || c.C != 2)) || (!ad.tracking && c.C != 1))
      throw std::runtime_error("dadaptive_step needs the rows `ad_m`, `vhat`, `ad_v` (amsgrad) and, with tracking, `ut` "
                               "and two published channels (one without)");
    check(consensus::launch_dadaptive_step<T>(ad, cur_stream()), "dadaptive_step");
  }
  void xg_check(const char* what) const {
    if (xg.xmix == nullptr || xg.theta_x == nullptr || xg.grad_part_x == nullptr || xg.g == nullptr ||
        xg.coef0 == nullptr || xg.coef == nullptr || c.sum_mode || c.C != 1 + c.dmax)
      throw std::runtime_error(std::string(what) + " needs the rows `xmix`, `theta_x`, `xg_g`, the cross partials "
                               "`grad_part_x`, the weights `xg_coef0` and `xg_coef`, the pointer-table neighbors and "
                               "one published channel per neighbor slot after the theta channel (C = 1 + dmax)");
  }
  void xg_pull() {
    xg_check("xg_pull");
    check(consensus::launch_xg_pull<T>(xg, cur_stream()), "xg_pull");
  }
  void xg_publish() {
    xg_check("xg_publish");
    check(consensus::launch_xg_publish<T>(xg, cur_stream()), "xg_publish");
  }
  void xg_step() {
    xg_check("xg_step");
    check(consensus::launch_xg_step<T>(xg, cur_stream()), "xg_step");
  }
  void relay_check(const char* what) const {
    if (rs.reach == nullptr || rs.rin == nullptr || rs.n < (T)1 || rs.diam < 0 || c.sum_mode || c.C != c.dmax)
      throw std::runtime_error(std::string(what) + " needs the reach table `reach`, the received rows `rin`, the node "
                               "count `relay_n`, the pointer-table neighbors and one published channel per neighbor "
                               "slot (C = dmax)");
  }
  void relay_mix() {
    relay_check("relay_mix");
    check(consensus::launch_relay_mix<T>(rs, cur_stream()), "relay_mix");
  }
  void relay_step() {
    relay_check("relay_step");
    check(consensus::launch_relay_step<T>(rs, cur_stream()), "relay_step");
  }
  void pg_check(const char* what) const {
    if (pg.seg == nullptr || pg.sign == nullptr || pg.nseg < 1 || (pg.vec == nullptr && pg.P + pg.Q > 0) ||
        pg.W < std::max(pg.P, pg.Q) + pg.B || c.sum_mode || c.C != c.dmax || c.dmax > consensus::kPgMaxDeg)
      throw std::runtime_error(std::string(what) + " needs the segment table `pg_seg` (`pg_nseg`, `pg_P`, `pg_Q`, `pg_B`), "
                               "the edge signs `pg_sign`, the vectors `pg_vec`, a message stride `pg_W` that holds both "
                               "phases, the pointer-table neighbors and one published channel per neighbor slot (C = "
                               "dmax <= " + std::to_string(consensus::kPgMaxDeg) + ")");
  }
  void pg_mix() {
    pg_check("pg_mix");
    check(consensus::launch_pg_mix<T>(pg, cur_stream()), "pg_mix");
  }
  void pg_step() {
    pg_check("pg_step");
    check(consensus::launch_pg_step<T>(pg, cur_stream()), "pg_step");
  }
  void cg_check(const char* what, bool clip) const {
    if (c.C != 1 || c.sum_mode)
      throw std::runtime_error(std::string(what) + " needs one published channel and the pointer-table neighbors");
    if (clip && (!cg_adaptive || cg.dist_part == nullptr || cg.pstride <= 0 || c.dmax > consensus::kClipMaxDeg))
      throw std::runtime_error(std::string(what) + " needs clip: adaptive, the distance partials `dist_part` with "
                               "`pstride` and at most " + std::to_string(consensus::kClipMaxDeg) + " neighbors per node");
    if (cg.attack != nullptr && cg.nbr_byz == nullptr)
      throw std::runtime_error(std::string(what) + " with attackers needs the Byzantine-neighbor table `nbr_byz`");
  }
  void cg_dist() {
    cg_check("cg_dist", true);
    check(consensus::launch_cg_dist<T>(cg, cur_stream()), "cg_dist");
  }
  void cg_mix() {
    cg_check("cg_mix", true);
    check(consensus::launch_cg_mix<T>(cg, cur_stream()), "cg_mix");
  }
  void cg_step() {
    cg_check("cg_step", false);
    check(consensus::launch_cg_step<T>(cg, cur_stream()), "cg_step");
  }
  void bridge_mix() {
    if (c.C != 1 || c.sum_mode || br.b < 0 || c.dmax > consensus::kBridgeMaxDeg)
      throw std::runtime_error("bridge_mix needs one published channel, the pointer-table neighbors, the screen "
                               "(`screen_b` >= 0, `screen_median`) and at most " +
                               std::to_string(consensus::kBridgeMaxDeg) + " neighbors per node");
    check(consensus::launch_bridge_mix<T>(br, cur_stream()), "bridge_mix");
  }
  void sgp_check(const char* what) const {
    if (sg.x == nullptr || sg.w == nullptr || sg.row_stride <= 0)
      throw std::runtime_error(std::string(what) + " needs the SGP rows `x`, `w` and `row_stride`");
  }
  void sgp_mix() {
    sgp_check("sgp_mix");
    check(consensus::launch_sgp_mix<T>(sg, cur_stream()), "sgp_mix");
  }
  void sgp_step() {
    sgp_check("sgp_step");
    check(consensus::launch_sgp_step<T>(sg, cur_stream()), "sgp_step");
  }
  void pdg_check(const char* what) const {
    if (pd.u == nullptr || pd.w == nullptr || pd.ysum == nullptr || pd.g_old == nullptr || pd.row_stride <= 0 || c.C != 2)
      throw std::runtime_error(std::string(what) + " needs the Push-DIGing rows `u`, `w`, `ysum`, `g_old`, `row_stride` "
                               "and two published channels");
  }
  void pdg_mix() {
    pdg_check("pdg_mix");
    check(consensus::launch_pdg_mix<T>(pd, cur_stream()), "pdg_mix");
  }
  void pdg_track() {
    pdg_check("pdg_track");
    check(consensus::launch_pdg_track<T>(pd, cur_stream()), "pdg_track");
  }
};

// local optimizer step of non-communicating nodes (solo / centralized baselines)
template <typename T>
struct LocalStepOp {
  consensus::LocalArgs<T> a{};
  explicit LocalStepOp(const py::dict& d) {
    a.c = common_from<T>(d);
    if (a.c.calls == nullptr) throw std::runtime_error("local_step needs the per-node step counter `calls`");
    a.m = ptr<T>(d, "m"); a.v = ptr<T>(d, "v");
    a.budget = ptr<const int>(d, "budget"); a.arrive = ptr<unsigned int>(d, "arrive");
    a.lr = (T)getf(d, "local_lr"); a.opt = geti(d, "opt", 1);
    if (a.budget == nullptr || a.arrive == nullptr) throw std::runtime_error("local_step needs `budget` and `arrive`");
    if (a.opt != consensus::kSGD && (a.m == nullptr || a.v == nullptr))
      throw std::runtime_error("local_step with Adam / AdamW needs the moment rows `m` and `v`");
  }
  void step() { check(consensus::launch_local_step<T>(a, cur_stream()), "local_step"); }
};

template <typename T>
static void bind_consensus(py::module& m, const char* name) {
  py::class_<ConsensusOp<T>>(m, name)
      .def(py::init<const py::dict&>())
      .def("dinno_update", &ConsensusOp<T>::dinno_update)
      .def("local_sum", &ConsensusOp<T>::local_sum)
      .def("dsgd_mix", &ConsensusOp<T>::dsgd_mix)
      .def("dsgd_step", &ConsensusOp<T>::dsgd_step)
      .def("dsgt_init", &ConsensusOp<T>::dsgt_init)
      .def("dsgt_mix", &ConsensusOp<T>::dsgt_mix)
      .def("dsgt_track", &ConsensusOp<T>::dsgt_track)
      .def("ed_mix", &ConsensusOp<T>::ed_mix)
      .def("ed_step", &ConsensusOp<T>::ed_step)
      .def("dsgdm_step", &ConsensusOp<T>::dsgdm_step)
      .def("choco_mix", &ConsensusOp<T>::choco_mix)
      .def("choco_step", &ConsensusOp<T>::choco_step)
      .def("beer_mix", &ConsensusOp<T>::beer_mix)
      .def("beer_step", &ConsensusOp<T>::beer_step)
      .def("kgt_mix", &ConsensusOp<T>::kgt_mix)
      .def("kgt_step", &ConsensusOp<T>::kgt_step)
      .def("ag_gossip", &ConsensusOp<T>::ag_gossip)
      .def("detag_track", &ConsensusOp<T>::detag_track)
      .def("hsgd_track", &ConsensusOp<T>::hsgd_track)
      .def("xg_pull", &ConsensusOp<T>::xg_pull)
      .def("xg_publish", &ConsensusOp<T>::xg_publish)
      .def("xg_step", &ConsensusOp<T>::xg_step)
      .def("pga_sum", &ConsensusOp<T>::pga_sum)
      .def("pga_mix", &ConsensusOp<T>::pga_mix)
      .def("slowmo_outer", &ConsensusOp<T>::slowmo_outer)
      .def("dp_norm", &ConsensusOp<T>::dp_norm)
      .def("dp_step", &ConsensusOp<T>::dp_step)
      .def("mq_mix", &ConsensusOp<T>::mq_mix)
      .def("mq_step", &ConsensusOp<T>::mq_step)
      .def("sparq_mix", &ConsensusOp<T>::sparq_mix)
      .def("sparq_step", &ConsensusOp<T>::sparq_step)
      .def("sparq_publish", &ConsensusOp<T>::sparq_publish)
      .def("dadaptive_mix", &ConsensusOp<T>::dadaptive_mix)
      .def("dadaptive_step", &ConsensusOp<T>::dadaptive_step)
      .def("relay_mix", &ConsensusOp<T>::relay_mix)
      .def("relay_step", &ConsensusOp<T>::relay_step)
      .def("pg_mix", &ConsensusOp<T>::pg_mix)
      .def("pg_step", &ConsensusOp<T>::pg_step)
      .def("cg_dist", &ConsensusOp<T>::cg_dist)
      .def("cg_mix", &ConsensusOp<T>::cg_mix)
      .def("cg_step", &ConsensusOp<T>::cg_step)
      .def("bridge_mix", &ConsensusOp<T>::bridge_mix)
      .def("sgp_mix", &ConsensusOp<T>::sgp_mix)
      .def("sgp_step", &ConsensusOp<T>::sgp_step)
      .def("pdg_mix", &ConsensusOp<T>::pdg_mix)
      .def("pdg_track", &ConsensusOp<T>::pdg_track);
}

void bind_mlp(py::module& m);     // mlp_bind.cpp
void bind_rl(py::module& m);      // rl_bind.cpp
void bind_runtime(py::module& m); // runtime.cpp

PYBIND11_MODULE(_C, m) {
  m.doc() = "nn_distributed_training_b200 sm_90a kernels";
  py::class_<MnistOp>(m, "MnistOp")
      .def(py::init<const py::dict&>())
      .def("update", &MnistOp::update)
      .def("train", &MnistOp::train)
      .def("eval", &MnistOp::eval);
  py::class_<GatherOp>(m, "GatherOp").def(py::init<const py::dict&>()).def("launch", &GatherOp::launch);
  m.def("debug_batch_indices", [](int mm, int B, int call, int seed, int node, uint64_t out, uint64_t out_size) {
    check(mnist::launch_batch_indices(mm, B, call, seed, node, reinterpret_cast<int*>(out),
                                      reinterpret_cast<int*>(out_size), cur_stream()), "batch_indices");
  });
  m.def("consensus_metric", [](bool f64, uint64_t rows, int N, int n_pad, int local0, int L, uint64_t inv_norm,
                               uint64_t out_pair, uint64_t out_mean) {
    auto r = reinterpret_cast<const int64_t*>(rows);
    auto a = reinterpret_cast<double*>(inv_norm); auto b = reinterpret_cast<double*>(out_pair); auto c = reinterpret_cast<double*>(out_mean);
    check(f64 ? consensus::launch_consensus_metric<double>(r, N, n_pad, local0, L, a, b, c, cur_stream())
              : consensus::launch_consensus_metric<float>(r, N, n_pad, local0, L, a, b, c, cur_stream()), "consensus_metric");
  });
  m.def("convnet_generic_smem_bytes", [](int F, int KS, int LW, int dtype64, int spb) {
    return (size_t)mnist::generic_smem_bytes(mnist::GenericShape{F, KS, LW, dtype64, 0.0, 1.0}, dtype64, spb);
  });
  m.def("convnet_generic_eval_spb", [](int F, int KS, int LW, int dtype64) {
    return mnist::generic_eval_spb(mnist::GenericShape{F, KS, LW, dtype64, 0.0, 1.0});
  });
  m.def("make_w1_tensor_map", [](uint64_t theta, int n_pad, int L, int off_w1) {
    unsigned char buf[128];
    check(mnist::make_w1_tensor_map(reinterpret_cast<const float*>(theta), n_pad, L, off_w1, buf), "make_w1_tensor_map");
    return py::bytes(reinterpret_cast<const char*>(buf), 128);
  });
  m.def("mnist_tc_max_clusters", []() { return mnist::tc_max_active_clusters(); });
  m.def("mnist_cl64_max_clusters", [](int nsplit) { return mnist::cl64_max_active_clusters(nsplit); }, py::arg("nsplit") = 1);
  m.def("mnist_cl64_cluster_ctas", []() { return mnist::cl64_cluster_ctas(); });
  m.def("rank_barrier", [](uint64_t slots, uint64_t peer_slot, int world, int rank, int epoch, uint64_t gate, uint64_t err) {
    check(consensus::launch_rank_barrier(reinterpret_cast<int*>(slots), reinterpret_cast<const int64_t*>(peer_slot), world, rank,
                                         epoch, reinterpret_cast<const volatile int*>(gate), reinterpret_cast<int*>(err), cur_stream()),
          "rank_barrier");
  });
  m.def("spin", [](long long cycles) { check(consensus::launch_spin(cycles, cur_stream()), "spin"); });
  bind_consensus<float>(m, "ConsensusOpF32");
  bind_consensus<double>(m, "ConsensusOpF64");
  py::class_<LocalStepOp<float>>(m, "LocalStepOpF32").def(py::init<const py::dict&>()).def("step", &LocalStepOp<float>::step);
  py::class_<LocalStepOp<double>>(m, "LocalStepOpF64").def(py::init<const py::dict&>()).def("step", &LocalStepOp<double>::step);
  bind_mlp(m);
  bind_rl(m);
  bind_runtime(m);
}
