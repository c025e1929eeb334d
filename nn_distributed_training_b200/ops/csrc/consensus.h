// Launch interface of the fused consensus kernels (consensus.cu).
//
// One launch covers every graph node hosted by this GPU.  Neighbor rows are read through a
// device pointer table, so a neighbor may be another row of the local arena (virtual nodes on
// one GPU) or a row of a peer GPU's symmetric-memory arena mapped over NVLink — the kernel is
// identical, the graph only changes which pointers are in the table.  All per-round scalars
// (rho_k, lr_k, alpha_k, graph id) are indexed by a device-side round counter so a captured
// CUDA graph can be replayed for any number of rounds with no host involvement.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nndt {
namespace consensus {

enum Opt : int { kSGD = 0, kAdam = 1, kAdamW = 2 };

template <typename T>
struct Common {
  // geometry
  int L, n_pad, S;            // local nodes, padded row length, gradient partials per node
  // live state (rows of the local arena)
  T* theta;                   // [L, n_pad]
  const T* grad_part;         // [L, S, n_pad]
  T* pub;                     // [2 parity, C chan, pub_L, n_pad] published rows (symmetric memory)
  int C, pub_L;
  // topology tables for G graphs
  const int64_t* nbr_ptr;     // [G, L, dmax, 2, C] device addresses of neighbor rows per parity/chan
  const T* nbr_w;             // [G, L, dmax]
  const T* self_w;            // [G, L]
  const int* deg;             // [G, L]
  const int* nbr_rank;        // [G, L, dmax] owning rank of each neighbor, -1 when local
  int dmax;
  // readers of each local node: the nodes that pull its row (its out-neighbors), which wait_neighbors also waits for.
  // rdr_deg == nullptr: every planned graph is undirected, the readers are the neighbors (deg, nbr_rank, dmax)
  const int* rdr_deg;         // [G, L] or nullptr
  const int* rdr_rank;        // [G, L, rmax] owning rank of each reader, -1 when local
  int rmax;
  // device-side schedules
  int* round_ctr;             // [1]
  const T* rho; const T* lr; const T* alpha;   // [oits]
  const int* graph_id;        // [oits]
  // sampler bookkeeping
  int* calls;                 // [L] or nullptr
  // optional device-side moving average of the training loss (online density metric, tloss_decay)
  const float* loss_part;     // [L, loss_S] per-CTA loss partials of the forward/backward kernel
  float* tloss;               // [L] tracker, nullptr = off
  float tdecay; int loss_S;
  // cross-GPU sync (nullptr / 0 when single GPU)
  int* flags;                 // [world] local slots written by peers (round published)
  const int64_t* peer_flag;   // [world] address of *their* slot for this rank
  int world, rank;
  unsigned long long notify_mask;  // ranks that ever own a neighbor of a local node: the only ones told about a new round
  const int* node_order;      // [L] launch order of the local nodes (nodes with remote neighbors first), nullptr = identity
  long long* timeline;        // debug (NNDT_TIMELINE=1): [4096][16] %globaltimer stamps of the update kernels, nullptr = off
  unsigned int* done_ctr;     // [1] last-block detection
  int* err;                   // [1] 1 = spin timeout, 2 = sequence check failed
  // optional debug build of the protocol (SURVEY 5.2): every published row carries the round it belongs to and every
  // neighbor read verifies it (nullptr = off)
  int* pub_seq;               // [2 parity, pub_L] local tags, written with the published rows
  const int64_t* nbr_seq;     // [G, L, dmax, 2] device addresses of the neighbors' tags per parity
  // complete-graph ("sum") mode: Metropolis weights are uniform 1/N, so every aggregate is a function of
  // S = sum over ALL nodes.  Each rank reduces its local rows into `sum_local` and the consumers fetch the
  // network-wide sum either with one NVLS in-switch reduction (multimem.ld_reduce over `sum_mc`) or, on a
  // single GPU, straight from `sum_local`.
  int sum_mode;               // 0 = pointer-table neighbors, 1 = complete graph via sums
  int n_total;                // N (all nodes of the graph)
  double* sum_local;          // [2 parity, C, n_pad] this rank's partial sums, always fp64: S - N theta_i cancels
  const double* sum_mc;       //   catastrophically in fp32 near consensus.  sum_mc = multicast mapping (or nullptr)
  int* sum_flags;             // [world] "partial sum of round k ready" flags written by peers
  const int64_t* peer_sum_flag;  // [world]
};

template <typename T>
struct DinnoArgs {
  Common<T> c;
  T* dual; T* delta; T* m; T* v;   // [L, n_pad]
  int step, pits, opt, persistent;
};

template <typename T>
struct DsgtArgs {
  Common<T> c;
  T* g_old;                        // [L, n_pad]
  // dsgt_mix variants (the distributed-PPO form): a per-coordinate step row instead of the alpha[k] schedule (constant
  // over rounds, 0 on the padding; nullptr = schedule), and the own-tracker step
  //   theta_i <- sum_j W_ij theta_j - alpha (.) y_i        (own_tracker = 1; y_i un-mixed)
  // instead of theta_i <- sum_j W_ij (theta_j - alpha y_j)
  const T* alpha_row;              // [n_pad] or nullptr
  int own_tracker;
};

// Exact Diffusion (Yuan, Ying, Zhao, Sayed 2019): DSGD's single published channel plus one local row psi.  The mix is
// DSGD's with the weights of A = (I + W) / 2 in the topology tables (complete-graph sum mode: (theta_i + S / N) / 2).
template <typename T>
struct EdArgs {
  Common<T> c;
  T* psi;                          // [L, n_pad] the adapt step of the previous round; set from theta in round 0
};

// DSGD with momentum: DSGD's single published channel and its mix (dsgd_mix_kernel), and a step that keeps a momentum
// row.  Local momentum: m is the heavy-ball row.  Quasi-global momentum (Lin, Karimireddy, Stich, Jaggi 2021; selected
// by x_prev != nullptr): m is mhat, the average of the rows' displacement (x_prev - x) / alpha_{k-1} over rounds, and
// x_prev the mixed row of the previous round.
template <typename T>
struct MomentumArgs {
  Common<T> c;
  T* m;                            // [L, n_pad] momentum (local) or mhat (quasi-global); read from round 1 on
  T* x_prev;                       // [L, n_pad] quasi-global: the previous round's mixed row; nullptr = local momentum
  T beta;                          // momentum coefficient, also mhat's averaging coefficient
  int nesterov;                    // step along g + beta m instead of m
};

// CHOCO-SGD (Koloskova, Stich, Jaggi 2019), memory-efficient form: nodes publish a compressed code of
// v = theta - x_hat instead of theta.  The published buffer holds code rows of `code_stride` bytes (nbr_ptr points at
// them); per block of 32 elements (b = i / 32, nb = n_pad / 32 blocks):
//   kCodeNone: [n_pad] T                          v itself
//   kCodeInt8: [n_pad] int8 codes, [nb] T scales  dec = code * scale, scale = max|v| / 127
//   kCodeSign: [nb] uint32 sign words, [nb] T     bit (i % 32) of word b set when v >= 0; dec = +-scale on live
//                                                 elements (bit set in `live`), 0 elsewhere; scale = sum|v| / n_live
//   kCodeTopk: [k] T values, [k] uint32 indices   the k = topk_k live elements of largest |v|, indices ascending, then
//                                                 zero padding to a multiple of 16 bytes (values first: fp64 values stay
//                                                 8-byte aligned for any k); dec = v at the indices (exact), 0 elsewhere.
//              Selection: keys are the IEEE bits of v with the sign bit cleared (+0 and -0 tie; the integer order is
//              the order of |v| in both dtypes), ordered by key descending, ties by the smaller index; the first k.
// The same layout is written by ops/consensus_ref.py: choco_encode / choco_decode.
enum Code : int { kCodeNone = 0, kCodeInt8 = 1, kCodeSign = 2, kCodeTopk = 3 };
// The top-k step selects with one thread-block cluster of kTopkCluster CTAs per node, each holding the v of its slice
// of the row (both channels for BEER) in shared memory: rows whose slices need more than kTopkRowSmem bytes are
// refused (ops/engine.py: check_topk_capacity)
constexpr int kTopkCluster = 8;
constexpr int kTopkRowSmem = 220 * 1024;

template <typename T>
struct ChocoArgs {
  Common<T> c;
  T* x_hat;                        // [L, n_pad] public estimate: the sum of the node's decoded codes
  T* s;                            // [L, n_pad] sum_j W_ij x_hat_j (own term included)
  const unsigned* live;            // [n_pad / 32] bit mask of the parameter elements (row padding and slot holes clear)
  T gamma;                         // consensus step
  int code;                        // Code
  long long code_stride;           // bytes per code row of the published buffer
  int topk_k;                      // entries of a kCodeTopk row
};

// BEER (Zhao, Li, Li, Richtárik, Chi 2022): DSGT's gradient tracking with both the parameters and the tracker gossiped
// through CHOCO's compressed differences.  Two published channels of CHOCO code rows (`code_stride` bytes, layout
// above): channel 0 the code of theta - h, channel 1 the code of v - g.
template <typename T>
struct BeerArgs {
  Common<T> c;
  T* h;                            // [L, n_pad] public estimate of theta: the sum of the node's decoded channel-0 codes
  T* s_h;                          // [L, n_pad] sum_j W_ij h_j (own term included)
  T* v;                            // [L, n_pad] gradient tracker
  T* g;                            // [L, n_pad] public estimate of v: the sum of the node's decoded channel-1 codes
  T* s_g;                          // [L, n_pad] sum_j W_ij g_j (own term included)
  T* m_old;                        // [L, n_pad] the gradient of the previous round
  const unsigned* live;            // [n_pad / 32] bit mask of the parameter elements
  T gamma;                         // consensus step
  int code;                        // Code
  long long code_stride;           // bytes per code row of the published buffer
  int topk_k;                      // entries of a kCodeTopk row
};

// K-GT (Liu, Lin, Koloskova, Stich 2023): gradient tracking with `K` local steps per communication round, and local
// DSGD (Koloskova et al. 2020) when `correction` is 0.  Correction mode publishes two channels, theta and y (the mean
// direction of the round's steps); local DSGD publishes theta only and mixes with dsgd_mix_kernel.  `step` is the
// index of the launch within the round, 0 .. K-1; the last one publishes.
template <typename T>
struct KgtArgs {
  Common<T> c;
  T* corr;                         // [L, n_pad] correction c_i, zero at the start (correction mode)
  T* dacc;                         // [L, n_pad] sum of the round's directions g + c; not read before step 0 writes it
  int step, K, correction;
};

// DeTAG (Lu, De Sa 2021): gradient tracking with K Chebyshev-accelerated gossip sub-steps per gradient step.  Channel 0
// of the published buffer is z = theta - alpha y, channel 1 the tracker y.  Every sub-step is a protocol round of its
// own: the device round counter counts sub-steps, p = K k + s, and `graph_id` / `alpha` hold K entries per gradient
// round.  `step` is the sub-step index s of the launch; the last one writes theta and `ymix` instead of publishing.
template <typename T>
struct DetagArgs {
  Common<T> c;
  const T* omega;                  // [K] the sub-step weights w_s (w_0 = 1)
  T* ymix;                         // [L, n_pad] Y_K of the last sub-step, read by detag_track (dead between rounds)
  T* g_old;                        // [L, n_pad] the gradient of the previous round (zero at the start)
  int step, K;
};

// GT-HSGD (Xin, Khan, Kar 2021): gradient tracking with a hybrid variance-reduced estimator, optimizers/gt_hsgd.py.
// The round is DSGT's (dsgt_mix first, channel 0 theta, channel 1 the tracker y) with a second forward/backward on
// the same minibatch at theta_prev; hsgd_track sums both partial sets (`c.grad_part` at theta, `grad_part_prev` at
// theta_prev, both with c.S rows per node), updates v and y, and stores theta_prev <- theta.
template <typename T>
struct HsgdArgs {
  Common<T> c;
  const T* grad_part_prev;         // [L, S, n_pad] partials of the forward/backward at theta_prev
  T* v;                            // [L, n_pad] the estimator v of the previous round (zero at the start)
  T* theta_prev;                   // [L, n_pad] the iterate of the previous round (theta^0 at the start)
  T omb;                           // 1 - beta, rounded once to T
};

// Cross-gradient gossip (CGA / NGC), optimizers/cross_gradient.py.  Gradient round k is two protocol rounds,
// p = 2k and p = 2k + 1, and the published buffer has C = 1 + dmax channels: channel 0 is the theta row, channel 1 + e
// node i's gradient at neighbor j_e's row.  The pointer-table entry of edge (i, e) for channel 1 + e names j_e's channel
// for i (its reverse slot), so the step pulls g_{j_e -> i}, the gradient node j_e took at theta_i.
//   xg_pull    (p = 2k):      xmix = sum_j W_ij theta_j and theta_x[e] = theta_{j_e} (the own row for e >= deg_i)
//   fwd/bwd at theta and at every theta_x[e], on one draw
//   xg_publish (p = 2k):      g = sum of the own partials; channel 1 + e of parity (p + 1) & 1 = sum of slot e's
//                             partials, e < deg_i; ends protocol round p
//   xg_step    (p = 2k + 1):  d = coef0 g + sum_e coef_e g_{j_e -> i} in fp64 (own term first, then table order),
//                             rounded once; theta = xmix - alpha d; publish theta into channel 0 of parity (p + 1) & 1
template <typename T>
struct XgArgs {
  Common<T> c;
  T* xmix;                         // [L, n_pad] the mixed row of the round (dead between rounds)
  T* theta_x;                      // [dmax, L, n_pad] the cross points of the round
  const T* grad_part_x;            // [dmax, L, S, n_pad] partials of the forward/backward at each cross point
  T* g;                            // [L, n_pad] the own gradient of the round
  const double* coef0;             // [G, L] (1 - lam) + lam W_ii
  const double* coef;              // [G, L, dmax] lam W_{i j_e}, 0 past deg_i
};

// Gossip-PGA (Chen, Yuan, Zhang, Pan, Xu, Yin 2021), optimizers/gossip_pga.py: DSGD's single published channel, with
// every `period`-th round (k mod period == period - 1) a global round that replaces the gossip mix with the exact
// network mean.  The round is pga_sum, pga_mix, fwd/bwd, dsgd_step; the branch is taken on the device from the round
// counter.  A global round reduces through the complete-graph fields of Common (sum_local, sum_mc, sum_flags,
// peer_sum_flag, n_total) while c.sum_mode stays 0, so gossip rounds pull through the pointer table.  The partial-sum
// buffer is indexed by the parity of the global round's count, (k / period) & 1 (consensus_device.cuh: pga_phase).
// `gossip` = 0 is local SGD: a gossip round leaves theta as it is and pulls nothing.
template <typename T>
struct PgaArgs {
  Common<T> c;
  int period;                      // >= 1
  int gossip;                      // 1 = Metropolis mix on gossip rounds, 0 = none (local SGD)
};

// SlowMo (Wang, Tantia, Ballas, Rabbat 2020), optimizers/slowmo.py: Gossip-PGA's round with an outer update after the
// global mix.  The round is pga_sum, pga_mix, slowmo_outer, fwd/bwd, then dsgd_step or (base momentum) dsgdm_step in
// local mode.  On a global round slowmo_outer takes xbar from theta (pga_mix wrote the mean there) and, in fp64 with
// gamma = alpha[k - 1] (alpha0 at k = 0),
//   u <- slow_momentum u + (anchor - xbar) / gamma;  anchor <- anchor - slow_lr gamma u;  theta <- anchor;  m <- 0
// rounding each stored row once; on a gossip round it returns at once.  It adds no cross-node traffic.
template <typename T>
struct SlowmoArgs {
  Common<T> c;
  T* anchor;                       // [L, n_pad] the point the last global round stepped to (theta^0 before it)
  T* u;                            // [L, n_pad] the slow momentum
  T* m;                            // [L, n_pad] the base momentum row zeroed on global rounds; nullptr = no base momentum
  int period;                      // >= 1, Gossip-PGA's
  T alpha0;                        // gamma of round 0
  double slow_lr, slow_momentum;
};

// DP-DSGD and DECOR (Allouah, Koloskova, El Mrini, Guerraoui, Jaggi 2024), optimizers/dp_dsgd.py: DSGD's single
// published channel and mix (dsgd_mix_kernel through the pointer table), then the node-level clipped and noised step
//   f_i = min(1, C / ||g_i||),  v_i = cz_dp xi_i + cz_pair sum_j s_ij xi_ij,  theta_i -= alpha_k (f_i g_i + v_i)
// dp_norm writes one fp64 partial of sum g^2 per chunk of THREADS * (16 / sizeof(T)) elements (as cg_dist), dp_step
// adds them in chunk order.  The normals come from Philox4x32-10 under `key` with the counter (element pair p, round k,
// a, b): (a, b) = (node, kDpLocal) for the node's own stream and (min(i, j), max(i, j)) for edge {i, j}, so both ends
// draw an edge's stream bit for bit; Box-Muller in fp64 gives elements 2p and 2p + 1 (ops/consensus_ref.py: dp_normals,
// the host twin).  v is evaluated in fp64, 0 off the live elements, and rounded once to T.
constexpr unsigned kDpLocal = 0xFFFFFFFFu;

template <typename T>
struct DpArgs {
  Common<T> c;
  double* norm_part;               // [L, pstride] partial sums of g^2, one per chunk
  int pstride;                     // >= the chunk count of a row
  const int* nbr_id;               // [G, L, dmax] global node id of each neighbor
  const unsigned* live;            // [n_pad / 32] live-element bits
  int node0;                       // global id of local node 0
  double clip;                     // C
  double cz_dp, cz_pair;           // C z_dp, C z_pair (both 0: no draw at all)
  unsigned key0, key1;             // Philox key
};

// Moniqua (Lu, De Sa 2020), optimizers/moniqua.py: modulo-quantized gossip on DSGD or Exact Diffusion.  The published
// buffer holds one code row per node of `code_stride` = n_pad * bits / 8 bytes: the bits-bit code of element e at bit
// (e * bits) % 32 of 32-bit word (e * bits) / 32.  With L = 2^bits and delta = 1 / L, in fp64:
//   encode  t = frac(x / B) L,  c = (floor(t) + (u < t - floor(t))) mod L,  u = r 2^-32
//   decode  v = y / B - c / L,  n = rint(v),  xhat = B (c / L + n)          y: the reader's own theta
// r is word e % 4 of Philox4x32-10 under `key` with the counter (e / 4, k, node, kMqTag): the code a node publishes for
// round k (written by the step of round k - 1), so a code depends on (seed, round, node, element, x) only.  Padding and
// slot holes (clear in `live`) get code 0.  Round k: mq_mix decodes the node's own code and its neighbors' against theta_i,
// theta_i += sum_{j != i} w_ij (xhat_j - xhat_i) in fp64 with the topology weights (W, or A = (I + W) / 2 for the Exact
// Diffusion base), rounded once; a neighbor element with |v - n| > 1/2 - delta is a margin hit, counted per node.
// mq_step takes DSGD's step (psi == nullptr) or ed_step's, encodes theta and publishes the code row
// (ops/consensus_ref.py: mq_mix_, mq_step_, the host twin).
constexpr unsigned kMqTag = 0x4D515244u;

template <typename T>
struct MoniquaArgs {
  Common<T> c;
  T* psi;                          // [L, n_pad] Exact Diffusion base: the adapt step of the previous round; nullptr = DSGD
  const unsigned* live;            // [n_pad / 32] live-element bits
  double B;                        // the modulus 2 theta_bound / (1 - 2 delta)
  int bits;                        // 2, 4 or 8
  unsigned key0, key1;             // Philox key
  int node0;                       // global id of local node 0
  unsigned long long* margin;      // [L] margin hits per local node
  long long code_stride;           // bytes per code row of the published buffer
};

// SPARQ-SGD (Singh, Data, George, Diggavi 2021), optimizers/sparq.py: CHOCO-SGD's compressed gossip with an event
// trigger and H local steps, on a fixed undirected graph.  A published row is a CHOCO code row (code_bytes, layout
// above, int8 / sign / none) followed by a 16-byte tail {uint32 trig, uint32 0, float64 e}: `row_stride` = code_bytes
// + 16.  Round k of node i:
//   sparq_mix:       s_i += sum over {i} u N_i with trig_j^{k-1} = 1 of W_ij dec(q_j), table order, own term first (a
//                    row whose tail says 0 is not read past its tail); theta_i += gamma (s_i - x_hat_i)
//   sparq_step(p):   theta_i -= alpha_k g_i, p = 0 .. H-1; the last step also writes the fp64 partials of
//                    (theta_i - x_hat_i)^2, one per chunk of THREADS * (16 / sizeof(T)) elements (dp_norm's chunks)
//   sparq_publish:   e_i = the partials summed in chunk order; trig = e_i > thr[k].  On a trigger q_i = Q(theta_i -
//                    x_hat_i) into parity (k+1) & 1 and x_hat_i += dec(q_i); either way the tail {trig, 0, e_i} and
//                    triggers[i] += trig
// (ops/consensus_ref.py: sparq_mix_, sparq_step_, sparq_publish_, the host twin).
template <typename T>
struct SparqArgs {
  Common<T> c;
  T* x_hat;                        // [L, n_pad] public estimate: the sum of the node's decoded codes
  T* s;                            // [L, n_pad] sum_j W_ij x_hat_j (own term included)
  const unsigned* live;            // [n_pad / 32] live-element bits
  const double* thr;               // [oits] trigger thresholds
  double* norm_part;               // [L, pstride] partial sums of (theta - x_hat)^2, one per chunk
  int pstride;                     // >= the chunk count of a row
  long long* triggers;             // [L] rounds each local node triggered in
  T gamma;                         // consensus step
  int code;                        // Code (none, int8, sign)
  long long code_bytes;            // bytes of the code part of a row
  long long row_stride;            // code_bytes + 16
  int step, H;                     // local step index of sparq_step, local steps per round
};

// Decentralized AMSGrad / AdaGrad (Chen, Karimi, Zhao, Li 2022), optimizers/dadaptive.py.  With `tracking` two published
// channels, theta and the second-moment tracker u~; the mix (dadaptive_mix_kernel) writes x into theta and
// z = sum_j W_ij u~_j into `ut`, the step turns z into the new u~ and publishes it without storing it back.  Without
// tracking one channel and dsgd_mix_kernel; the step divides by the node's own vhat.
template <typename T>
struct DAdaptiveArgs {
  Common<T> c;
  T* m;                            // [L, n_pad] first moment, zero at the start
  T* v;                            // [L, n_pad] amsgrad: second moment, zero at the start; nullptr with adagrad
  T* vhat;                         // [L, n_pad] amsgrad: max of v; adagrad: running mean of g^2.  eps at the start
  T* ut;                           // [L, n_pad] tracking: z of the round's mix (read by the step); nullptr = own vhat
  T beta1, beta2, eps;
  int adagrad, tracking;
};

// RelaySum (Vogels et al. 2021), optimizers/relaysum.py, on a fixed tree.  The published buffer has C = dmax channels:
// channel e of node i is its message m_{i -> j_e} for its e-th neighbor.  The pointer table's channel-0 entry of edge
// (i, e) names neighbor j_e's channel for i (its reverse slot), so a round pulls one row per edge, as DSGD's.  relay_mix
// keeps the deg received rows in `rin` and writes x into theta; relay_step writes h into theta and publishes the deg
// messages h + sum_{e' != e} r_e' into the other parity.  The step holds the received rows in registers, so a node
// has at most kRelayMaxDeg neighbors (ops/engine.py: check_relay_plan).
constexpr int kRelayMaxDeg = 16;

template <typename T>
struct RelayArgs {
  Common<T> c;
  const T* reach;                  // [L, diam + 1] R_i^k - 1 (exact in T), read at min(k, diam)
  T* rin;                          // [L, dmax, n_pad] the messages received in the round's mix
  int diam;
  T n;                             // nodes of the tree
};

// PowerGossip (Vogels, Karimireddy, Jaggi 2020), optimizers/powergossip.py, on a fixed undirected graph.  Round k runs
// phase k & 1.  The published buffer has C = dmax channels of message rows `W` elements long (not n_pad): channel e of
// node i is its message for neighbor j_e, [per matrix the product h q (phase 0, m_l long) or h^T p (phase 1, n_l long) |
// the 1-D tensors (B)], and the pointer table's channel-0 entry of edge (i, e) names j_e's channel for i, as RelaySum's.
// pg_mix pulls the deg messages into shared memory as canonical differences d = a_lo - a_hi, writes
// x = h - gamma sum_e W_ie s_ie U_e into theta and the next vectors d / |d| into `vec` (|d| in fp64, one fixed order);
// pg_step writes h into theta and publishes the products of phase (k + 1) & 1 into the other parity.
// Segment s of `seg` is one parameter tensor in slot order: {offset, m, n, poff, qoff}, n = 0 for a 1-D tensor (m its
// length, poff its offset in the bias block).  A node has at most kPgMaxDeg neighbors, and its deg message differences
// must fit the opt-in shared memory (ops/engine.py: check_powergossip_capacity).
constexpr int kPgMaxDeg = 16;
constexpr int kPgVecChunk = 256;   // elements of a 1-D tensor one warp of pg_step publishes per unit

template <typename T>
struct PgArgs {
  Common<T> c;
  T* vec;                          // [L, dmax, P + Q] every edge's p (row space) then q (column space)
  const int* seg;                  // [nseg, 5]
  const int* sign;                 // [L, dmax] +1 when this node is the edge's lower endpoint, else -1
  int nseg, P, Q, B, W;            // segments, sum m, sum n, bias elements, message row stride (elements)
  T gamma;
  int grid_x;                      // CTAs per node, 0 = one wave (the messages do not depend on it)
};

// ClippedGossip (He, Karimireddy, Jaggi 2022): DSGD's single published channel with a self-centred clipped mix, and
// Byzantine nodes that publish an attack row instead of theta.  Round k: cg_dist reduces the squared
// distances |theta_j^pub - theta_i|^2 of every neighbor, one partial per fixed chunk of the row, into dist_part; cg_mix
// sums the partials in chunk order (every CTA of a node gets the same distances), picks the radius tau_i and mixes
//   theta_i <- theta_i + sum_j W_ij min(1, tau_i / d_ij) (theta_j^pub - theta_i);
// cg_step is dsgd_step, and a Byzantine node publishes -scale theta_i (sign flip) or mu - z sigma of its honest
// neighbors' rows of round k (ALIE) in place of theta_i.
enum Attack : int { kHonest = 0, kSignFlip = 1, kAlie = 2 };
constexpr int kClipMaxDeg = 128;   // neighbors per node cg_mix sorts in shared memory
// a prefix of weights fits in delta up to this slack: the weights of an fp32 table are rounded (1/10 becomes
// 0.100000001), and two of them must still fit in delta = 0.2
constexpr double kClipSlack = 1e-6;

template <typename T>
struct ClipArgs {
  Common<T> c;
  double* dist_part;               // [L, dmax, pstride] partial sums of the squared distances, one per chunk of
                                   // THREADS * (16 / sizeof(T)) elements of the row
  int pstride;                     // >= the chunk count of a row
  const int* attack;               // [L] Attack code of each local node, nullptr = no attacker on this rank
  const int* nbr_byz;              // [G, L, dmax] 1 when the neighbor is Byzantine (ALIE averages the others)
  double delta;                    // Metropolis weight of the neighbors that may be clipped
  double scale, z;                 // sign-flip scale, ALIE's z
};

// BRIDGE (Fang, Yang, Bajwa 2022), optimizers/bridge.py: DSGD's single published channel with a coordinate-wise
// screened mix, and ClippedGossip's step and attack rows (cg_step with a ClipArgs).  Per element, bridge_mix sorts the
// deg neighbor values of round k and writes into theta
//   trimmed mean: (theta_i + sorted positions [b, deg - b), ascending) / (1 + max(0, deg - 2b))
//   median:       the median of theta_i and the deg values, 0.5 (lower + upper) of an even count
// summed and averaged in fp64 and rounded once.  The neighbor values sit in registers: a node has at most
// kBridgeMaxDeg neighbors (ops/engine.py: check_bridge_capacity).
constexpr int kBridgeMaxDeg = 16;

template <typename T>
struct ScreenArgs {
  Common<T> c;
  int b;                           // values trimmed at each end (trimmed mean)
  int median;                      // 1 = median screen, 0 = trimmed mean
};

// SGP, Stochastic Gradient Push (Assran et al. 2019): push-sum gossip over a column-stochastic A, on directed graphs.
// The topology tables hold in-neighbors (nbr_ptr, deg, nbr_rank) and the weights of A (nbr_w = A_ij, self_w = A_ii).
// A published row is [n_pad] T numerators x, then a 16-byte tail whose first 8 bytes are the float64 push-sum weight w:
// `row_stride` = n_pad * sizeof(T) + 16 bytes.  theta = x / w is the de-biased row the forward/backward kernel reads.
// A plan with a directed graph carries reader tables (Common::rdr_deg): the round-start wait covers the out-neighbors.
template <typename T>
struct SgpArgs {
  Common<T> c;
  T* x;                            // [L, n_pad] numerators
  double* w;                       // [L] push-sum weights
  long long row_stride;            // bytes per published row
};

// Push-DIGing (Nedić, Olshevsky, Shi 2017): DSGT's gradient tracking on push-sum gossip, for directed and time-varying
// graphs.  The topology tables are SGP's (in-neighbors, A = push weights).  Two published channels, each row of
// `row_stride` = n_pad * sizeof(T) + 16 bytes: channel 0 holds the numerators u with the float64 push-sum weight w in
// its tail, channel 1 the tracker y (its tail is never read).  theta = u / w is the row the forward/backward kernel reads.
template <typename T>
struct PushDigArgs {
  Common<T> c;
  T* u;                            // [L, n_pad] numerators
  double* w;                       // [L] push-sum weights
  T* ysum;                         // [L, n_pad] sum_j A_ij y_j^pub of the round (own term included)
  T* g_old;                        // [L, n_pad] the gradient of the previous round
  long long row_stride;            // bytes per published row
};

// Local optimizer step of nodes that do not communicate (solo and centralized baselines): per node, the gradient
// partials are summed and one torch.optim SGD / Adam / AdamW step is applied, while c.calls[l] < budget[l].
// Uses c.L, c.n_pad, c.S, c.theta, c.grad_part and c.calls (the node's step counter, required).
template <typename T>
struct LocalArgs {
  Common<T> c;
  T* m; T* v;                      // [L, n_pad] moments (nullptr with SGD)
  const int* budget;               // [L] steps each node takes in all
  unsigned int* arrive;            // [L] CTA arrival counters: calls[l] advances once every CTA of node l has read it
  T lr;
  int opt;
};

template <typename T> cudaError_t launch_local_step(const LocalArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_dinno_update(const DinnoArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_dsgd_mix(const Common<T>& c, cudaStream_t st);
template <typename T> cudaError_t launch_dsgd_step(const Common<T>& c, cudaStream_t st);
template <typename T> cudaError_t launch_dsgt_init(const DsgtArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_dsgt_mix(const DsgtArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_dsgt_track(const DsgtArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_ed_mix(const EdArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_ed_step(const EdArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_dsgdm_step(const MomentumArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_choco_mix(const ChocoArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_choco_step(const ChocoArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_beer_mix(const BeerArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_beer_step(const BeerArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_kgt_mix(const KgtArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_kgt_step(const KgtArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_ag_gossip(const DetagArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_detag_track(const DetagArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_hsgd_track(const HsgdArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_xg_pull(const XgArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_xg_publish(const XgArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_xg_step(const XgArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_pga_sum(const PgaArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_pga_mix(const PgaArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_slowmo_outer(const SlowmoArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_dp_norm(const DpArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_dp_step(const DpArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_mq_mix(const MoniquaArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_mq_step(const MoniquaArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_sparq_mix(const SparqArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_sparq_step(const SparqArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_sparq_publish(const SparqArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_dadaptive_mix(const DAdaptiveArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_dadaptive_step(const DAdaptiveArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_relay_mix(const RelayArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_relay_step(const RelayArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_pg_mix(const PgArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_pg_step(const PgArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_cg_dist(const ClipArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_cg_mix(const ClipArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_cg_step(const ClipArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_bridge_mix(const ScreenArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_sgp_mix(const SgpArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_sgp_step(const SgpArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_pdg_mix(const PushDigArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_pdg_track(const PushDigArgs<T>& a, cudaStream_t st);
template <typename T> cudaError_t launch_local_sum(const Common<T>& c, cudaStream_t st);

// All-rank barrier on the device (bench start alignment, metric quiescence): every rank stores `epoch` into its slot of
// every peer's array and spins until all of its own slots reached it; with `gate` != nullptr the kernel first spins on that
// (pinned host) word until the host sets it, so everything enqueued behind it starts at the host's command.
cudaError_t launch_rank_barrier(int* slots, const int64_t* peer_slot, int world, int rank, int epoch,
                                const volatile int* gate, int* err, cudaStream_t st);
// Busy-wait `cycles` SM clocks (tests: a deliberately delayed rank)
cudaError_t launch_spin(long long cycles, cudaStream_t st);

// K6 consensus metric (problems/dist_mnist_problem.py:155-169): distances between L2-normalised parameter rows.
// rows[j] is the device address of node j's current row (local, or a peer GPU's published row over NVLink).
// out_pair [L, N] = |th_i/|th_i| - th_j/|th_j||,  out_mean [L] = |th_i/|th_i| - mean_j th_j/|th_j||   (fp64 accumulation)
template <typename T>
cudaError_t launch_consensus_metric(const int64_t* rows, int N, int n_pad, int local0, int L, double* inv_norm,
                                    double* out_pair, double* out_mean, cudaStream_t st);

}  // namespace consensus
}  // namespace nndt
