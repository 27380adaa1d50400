// Engine: checkpoint packing, device arena and the launch sequence of the hot path.
// Reference call stack being replaced: inference.py:70-102 (Separator.separate / separate_tta) ->
// inference.py:42-68 (_separate) -> lib/nets.py:124-131 (predict_mask) -> lib/nets.py:82-117 (forward)
// -> lib/nets.py:26-41 (BaseNet) -> lib/layers.py.
#include "engine.h"
#include "tc_plan.h"

#include <math.h>
#include <stdio.h>
#include <string.h>

namespace vr {

static const double kBnEps = 1e-5;   // nn.BatchNorm2d / BatchNorm1d default eps

bool Engine::ck(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return true;
  err = std::string(what) + ": " + cudaGetErrorString(e);
  return false;
}

bool upload(void* dst, const void* src, size_t bytes, std::string& err) {
  const cudaError_t e = cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) return true;
  err = std::string("cudaMemcpy(") + std::to_string(bytes) + ", host to device): " + cudaGetErrorString(e);
  return false;
}

void* Engine::dalloc(Arena& arena, size_t bytes, const void* host) {
  const size_t n = bytes == 0 ? 16 : bytes;
  DevPtr<void> m;
  const cudaError_t e = m.alloc(n);
  if (e != cudaSuccess) {
    err = std::string("cudaMalloc(") + std::to_string(n) + "): " + cudaGetErrorString(e);
    return nullptr;
  }
  // pad channels must be finite zeros forever (zero weights multiply them)
  if (!ck(cudaMemset(m.get(), 0, n), "cudaMemset")) return nullptr;
  if (host && !upload(m.get(), host, bytes, err)) return nullptr;
  arena.push_back(std::move(m));
  return arena.back().get();
}

Buffer Engine::make_buffer(Arena& arena, int N, int H, int W, int C, int pad_w) {
  Buffer b;
  b.N = N; b.H = H; b.W = W; b.C = C;
  b.Wp = W + pad_w;
  size_t plane = (size_t)N * H * b.Wp * C * sizeof(bf16);
  plane = (plane + 1023) / 1024 * 1024;
  char* p = (char*)dalloc(arena, 2 * plane);
  if (p) {
    b.hi = (bf16*)p;
    b.lo = (bf16*)(p + plane);
  }
  return b;
}

Engine::Engine(const Config& cfg) : cfg_(cfg) {
  if (cudaSetDevice(cfg_.device) != cudaSuccess) {
    err = "cudaSetDevice failed (no CUDA device? this library has no CPU path)";
    return;
  }
  const int NF = cfg_.n_fft;
  std::vector<float2> tw(NF / 2);
  std::vector<float> win(NF);
  for (int q = 0; q < NF / 2; ++q) {
    double a = -2.0 * M_PI * (double)q / (double)NF;
    tw[q] = make_float2((float)cos(a), (float)sin(a));
  }
  for (int n = 0; n < NF; ++n) win[n] = (float)(0.5 - 0.5 * cos(2.0 * M_PI * (double)n / (double)NF));
  twiddle_ = (float2*)dalloc(arena_, sizeof(float2) * tw.size(), tw.data());
  window_ = (float*)dalloc(arena_, sizeof(float) * win.size(), win.data());
  ws_norm_ = (float*)dalloc(arena_, sizeof(float) * 4);
  ws_lex_ = (unsigned long long*)dalloc(arena_, sizeof(unsigned long long));
  if (!twiddle_ || !window_ || !ws_norm_ || !ws_lex_) return;
  cudaStreamCreateWithFlags(&s_hi_, cudaStreamNonBlocking);
  cudaStreamCreateWithFlags(&s_copy_, cudaStreamNonBlocking);
  cudaEventCreateWithFlags(&ev_span_, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&ev_fork_, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&ev_join_, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&ev_lstm_fork_, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&ev_lstm_join_, cudaEventDisableTiming);
}

// the members that own device memory are destroyed after this body, with the context's device current
Engine::~Engine() {
  cudaSetDevice(cfg_.device);
  profile_enable(false);
  if (s_hi_) cudaStreamDestroy(s_hi_);
  if (s_copy_) cudaStreamDestroy(s_copy_);
  if (ev_span_) cudaEventDestroy(ev_span_);
  if (ev_fork_) cudaEventDestroy(ev_fork_);
  if (ev_join_) cudaEventDestroy(ev_join_);
  if (ev_lstm_fork_) cudaEventDestroy(ev_lstm_fork_);
  if (ev_lstm_join_) cudaEventDestroy(ev_lstm_join_);
}

bool Engine::load_tensor(const char* name, int dtype, int ndim, const int64_t* shape, const void* data) {
  HostTensor t;
  int64_t n = 1;
  for (int i = 0; i < ndim; ++i) {
    t.shape.push_back(shape[i]);
    n *= shape[i];
  }
  t.data.resize((size_t)n);
  if (dtype == 0) {
    memcpy(t.data.data(), data, sizeof(float) * (size_t)n);
  } else if (dtype == 1) {   // int64 (BatchNorm num_batches_tracked): kept only for strict key checking
    const int64_t* p = (const int64_t*)data;
    for (int64_t i = 0; i < n; ++i) t.data[(size_t)i] = (float)p[i];
  } else {
    err = std::string("unsupported dtype for tensor ") + name;
    return false;
  }
  sd_[name] = std::move(t);
  finalized_ = false;
  return true;
}

bool Engine::need(const std::string& key, std::initializer_list<int64_t> shape, const HostTensor** out) {
  auto it = sd_.find(key);
  if (it == sd_.end()) {
    err = "missing key in state_dict: " + key;
    return false;
  }
  std::vector<int64_t> s(shape);
  if (it->second.shape != s) {
    std::string got, want;
    for (auto d : it->second.shape) got += std::to_string(d) + ",";
    for (auto d : s) want += std::to_string(d) + ",";
    err = "size mismatch for " + key + ": checkpoint (" + got + ") vs model (" + want + ")";
    return false;
  }
  *out = &it->second;
  return true;
}

bool Engine::fold_bn(const std::string& bn, int C, const float* pre_bias, std::vector<double>& scale,
                     std::vector<double>& shift) {
  const HostTensor *g, *b, *m, *v, *cnt;
  if (!need(bn + ".weight", {C}, &g) || !need(bn + ".bias", {C}, &b) || !need(bn + ".running_mean", {C}, &m) ||
      !need(bn + ".running_var", {C}, &v) || !need(bn + ".num_batches_tracked", {}, &cnt))
    return false;
  scale.resize((size_t)C);
  shift.resize((size_t)C);
  for (int c = 0; c < C; ++c) {
    scale[(size_t)c] = (double)g->data[(size_t)c] / sqrt((double)v->data[(size_t)c] + kBnEps);
    shift[(size_t)c] = scale[(size_t)c] * ((pre_bias ? (double)pre_bias[c] : 0.0) - (double)m->data[(size_t)c]) +
                       (double)b->data[(size_t)c];
  }
  return true;
}

// Packs OIHW weights w [Cout][Cin][L.k][L.k], output channel co times scale[co] (in double, rounded to float once), to
// wp [tap][CinPad][CoutPad] with CinPad = perm.size(): packed input channel pc holds channel perm[pc], or zeros where
// that is -1.  bp [CoutPad] is shift rounded to float.  Sets L's channel counts.
static void pack_conv(ConvLayer& L, const float* w, int Cout, int Cin, const double* scale, const double* shift,
                      const std::vector<int>& perm, std::vector<float>& wp, std::vector<float>& bp) {
  L.Cin = Cin; L.CinPad = (int)perm.size(); L.Cout = Cout; L.CoutPad = round_up(Cout, 8);
  const int taps = L.k * L.k;
  wp.assign((size_t)taps * L.CinPad * L.CoutPad, 0.f);
  bp.assign((size_t)L.CoutPad, 0.f);
  for (int co = 0; co < Cout; ++co) {
    bp[(size_t)co] = (float)shift[co];
    for (int pc = 0; pc < L.CinPad; ++pc) {
      const int ci = perm[(size_t)pc];
      if (ci < 0) continue;
      for (int t = 0; t < taps; ++t)
        wp[((size_t)t * L.CinPad + pc) * L.CoutPad + co] =
            (float)((double)w[((size_t)co * Cin + ci) * taps + t] * scale[co]);
    }
  }
}

bool Engine::prepare_conv(ConvLayer& L, Arena& arena, const std::vector<float>& wp, const std::vector<float>& bp,
                          bool use_tc, int H, int W, bool rows_wide) {
  if (use_tc && !tc_prepare(L, wp.data(), bp.data(), H, W, rows_wide, err)) return false;
  if (L.tc) return true;
  L.w = (float*)dalloc(arena, wp.size() * sizeof(float), wp.data());
  L.bias = (float*)dalloc(arena, bp.size() * sizeof(float), bp.data());
  return L.w && L.bias;
}

// Fold BatchNorm2d(eval) into the bias-free conv (lib/layers.py:12-23) and prepare it for its kernel.
// perm[packed_ci] = original input channel, or -1 for a zero (padding) channel.
bool Engine::make_conv(ConvLayer& L, const std::string& prefix, const std::vector<int>& perm, int k, int stride,
                       int dh, int dw, int act, int H, int W, bool rows_wide) {
  L.name = prefix;
  L.k = k; L.stride = stride; L.dil_h = dh; L.dil_w = dw; L.act = act;
  auto itw = sd_.find(prefix + ".conv.0.weight");
  if (itw == sd_.end()) {
    err = "missing key in state_dict: " + prefix + ".conv.0.weight";
    return false;
  }
  const HostTensor& w = itw->second;
  if (w.shape.size() != 4 || w.shape[2] != k || w.shape[3] != k) {
    err = "size mismatch for " + prefix + ".conv.0.weight";
    return false;
  }
  const int Cout = (int)w.shape[0], Cin = (int)w.shape[1];
  int used = 0;
  for (int v : perm) used += v >= 0;
  if (used != Cin) {
    err = "internal: channel permutation does not cover the input channels of " + prefix;
    return false;
  }
  std::vector<double> scale, shift;
  if (!fold_bn(prefix + ".conv.1", Cout, nullptr, scale, shift)) return false;
  std::vector<float> wp, bp;
  pack_conv(L, w.data.data(), Cout, Cin, scale.data(), shift.data(), perm, wp, bp);
  return prepare_conv(L, arena_, wp, bp, cfg_.conv_mode == 0, H, W, rows_wide);
}

static std::vector<int> identity_perm(int c, int pad) {
  std::vector<int> p((size_t)pad, -1);
  for (int i = 0; i < c; ++i) p[(size_t)i] = i;
  return p;
}

bool Engine::build_basenet(BaseNetPlan& P, const std::string& prefix, const std::vector<int>& in_perm, int n, int H,
                           int W, int nin_lstm, int nout_lstm) {
  P.prefix = prefix; P.n = n; P.H = H; P.W = W;
  const int Nb = cfg_.max_batch;
  if (H % 16 || W % 16 || n % 4) {
    err = "unsupported geometry: band height and cropsize must be multiples of 16 and nout a multiple of 16";
    return false;
  }
  if (!make_conv(P.enc1, prefix + ".enc1", in_perm, 3, 1, 1, 1, ACT_RELU, H, W)) return false;
  const int mult[5] = {1, 2, 4, 6, 8};
  for (int i = 0; i < 4; ++i) {
    const int cin = n * mult[i], cout = n * mult[i + 1], Ho = H >> (i + 1), Wo = W >> (i + 1);
    const std::string e = prefix + ".enc" + std::to_string(i + 2);
    if (!make_conv(P.enc_a[i], e + ".conv1", identity_perm(cin, round_up(cin, 8)), 3, 2, 1, 1, ACT_LEAKY, Ho, Wo))
      return false;
    if (!make_conv(P.enc_b[i], e + ".conv2", identity_perm(cout, cout), 3, 1, 1, 1, ACT_LEAKY, Ho, Wo)) return false;
  }
  const int c8 = 8 * n, h16 = H / 16, w16 = W / 16;
  if (!make_conv(P.aspp1, prefix + ".aspp.conv1.1", identity_perm(c8, c8), 1, 1, 1, 1, ACT_RELU, 1, w16))
    return false;
  if (!make_conv(P.aspp2, prefix + ".aspp.conv2", identity_perm(c8, c8), 1, 1, 1, 1, ACT_RELU, h16, w16))
    return false;
  const int dil[3][2] = {{4, 2}, {8, 4}, {12, 6}};   // lib/nets.py:10
  for (int i = 0; i < 3; ++i)
    if (!make_conv(P.aspp_d[i], prefix + ".aspp.conv" + std::to_string(i + 3), identity_perm(c8, c8), 3, 1,
                   dil[i][0], dil[i][1], ACT_RELU, h16, w16))
      return false;
  if (!make_conv(P.bott, prefix + ".aspp.bottleneck", identity_perm(5 * c8, 5 * c8), 1, 1, 1, 1, ACT_RELU, h16, w16))
    return false;
  if (!make_conv(P.dec[0], prefix + ".dec4.conv1", identity_perm(14 * n, 14 * n), 3, 1, 1, 1, ACT_RELU, H / 8, W / 8))
    return false;
  if (!make_conv(P.dec[1], prefix + ".dec3.conv1", identity_perm(10 * n, 10 * n), 3, 1, 1, 1, ACT_RELU, H / 4, W / 4))
    return false;
  // rows_wide: dec2's upsample is fused into the row kernel whenever 4n is a multiple of 32
  if (!make_conv(P.dec[2], prefix + ".dec2.conv1", identity_perm(6 * n, 6 * n), 3, 1, 1, 1, ACT_RELU, H / 2, W / 2,
                 true))
    return false;
  // dec1 input in the reference: cat[ up(cat[h (2n), lstm (1)]) , e1 (n) ]  (lib/nets.py:38-39, layers.py:52-56),
  // reduced as [ up(h) 2n | zeros up to Up | e1 n | zeros up to Lp | up(lstm) 1 | 15 zeros ] (BaseNetPlan, engine.h)
  const int lg = 16;   // the lstm channel + 15 zeros keep every slice 32-byte aligned (full-sector 256-bit stores)
  const int Up = round_up(2 * n, 32), Lp = round_up(Up + n, 16), c1 = Lp + lg;
  {
    std::vector<int> perm((size_t)c1, -1);
    for (int i = 0; i < 2 * n; ++i) perm[(size_t)i] = i;
    for (int i = 0; i < n; ++i) perm[(size_t)(Up + i)] = 2 * n + 1 + i;
    perm[(size_t)Lp] = 2 * n;
    // (the 64-wide tile was measured on dec1 as well - one N tile instead of two for n = 64 - and is no faster there:
    //  with its single accumulator set the epilogue no longer overlaps the next tile's products)
    if (!make_conv(P.dec[3], prefix + ".dec1.conv1", perm, 3, 1, 1, 1, ACT_RELU, H, W)) return false;
  }

  // activation buffers: the decoders' plans decide what their concat buffers hold
  P.fused2 = P.dec[2].tc && P.dec[2].tc->fuses_upsample(4 * n);
  P.fused1 = P.dec[3].tc && P.dec[3].tc->fuses_upsample(Up);
  P.dot2 = P.dec[2].tc && P.dec[2].tc->fuses_dot();
  P.lstm_own = P.fused1 && n % 32 == 0;
  const int c1_first = P.fused1 ? Up : 0;   // the first of dec1's reduction channels that cat1 holds
  P.lstm_coff = Lp - c1_first;
  P.cat1 = make_buffer(arena_, Nb, H, W, (P.lstm_own ? Lp : c1) - c1_first);
  if (P.lstm_own) P.lstm_up = make_buffer(arena_, Nb, H, W, 8);
  P.t2 = make_buffer(arena_, Nb, H / 2, W / 2, 2 * n);
  P.cat2 = make_buffer(arena_, Nb, H / 2, W / 2, P.fused2 ? 2 * n : 6 * n);
  P.t3 = make_buffer(arena_, Nb, H / 4, W / 4, 4 * n);
  P.cat3 = make_buffer(arena_, Nb, H / 4, W / 4, 10 * n);
  P.t4 = make_buffer(arena_, Nb, H / 8, W / 8, 6 * n);
  P.cat4 = make_buffer(arena_, Nb, H / 8, W / 8, 14 * n);
  P.t5 = make_buffer(arena_, Nb, H / 16, W / 16, 8 * n);
  P.e5 = make_buffer(arena_, Nb, H / 16, W / 16, 8 * n);
  P.pool = make_buffer(arena_, Nb, 1, W / 16, 8 * n);
  P.f1 = make_buffer(arena_, Nb, 1, W / 16, 8 * n);
  P.acat = make_buffer(arena_, Nb, H / 16, W / 16, 40 * n);
  P.ao = make_buffer(arena_, Nb, H / 16, W / 16, 8 * n);
  P.d4 = make_buffer(arena_, Nb, H / 8, W / 8, 6 * n);
  P.d3 = make_buffer(arena_, Nb, H / 4, W / 4, 4 * n);
  P.d2 = make_buffer(arena_, Nb, H / 2, W / 2, Up);
  if (!P.d2.hi || !P.cat1.hi) return false;

  // ---- LSTM module (lib/layers.py:110-122) ----
  LstmPlan& Q = P.lstm;
  const std::string lp = prefix + ".lstm_dec2";
  Q.C = 2 * n; Q.bins = H / 2; Q.T = W / 2; Q.hid = nout_lstm / 2;
  if (Q.bins != nin_lstm) {
    err = "LSTM input size does not match band height / 2 for " + lp;
    return false;
  }
  const HostTensor* cw;
  std::vector<double> scale, shift;
  if (!need(lp + ".conv.conv.0.weight", {1, Q.C, 1, 1}, &cw) ||
      !fold_bn(lp + ".conv.conv.1", 1, nullptr, scale, shift))
    return false;
  {
    std::vector<float> w((size_t)Q.C);
    for (int c = 0; c < Q.C; ++c) w[(size_t)c] = (float)((double)cw->data[(size_t)c] * scale[0]);
    Q.conv_bias = (float)shift[0];
    Q.conv_w = (float*)dalloc(arena_, sizeof(float) * w.size(), w.data());
    if (!Q.conv_w) return false;
  }
  {
    const int H4 = 4 * Q.hid;
    std::vector<float> wih((size_t)2 * H4 * Q.bins), bih((size_t)2 * H4), whh((size_t)2 * H4 * Q.hid);
    const char* sfx[2] = {"", "_reverse"};
    for (int d = 0; d < 2; ++d) {
      const HostTensor *a, *h, *b1, *b2;
      if (!need(lp + ".lstm.weight_ih_l0" + sfx[d], {H4, Q.bins}, &a) ||
          !need(lp + ".lstm.weight_hh_l0" + sfx[d], {H4, Q.hid}, &h) ||
          !need(lp + ".lstm.bias_ih_l0" + sfx[d], {H4}, &b1) || !need(lp + ".lstm.bias_hh_l0" + sfx[d], {H4}, &b2))
        return false;
      memcpy(&wih[(size_t)d * H4 * Q.bins], a->data.data(), sizeof(float) * (size_t)H4 * Q.bins);
      memcpy(&whh[(size_t)d * H4 * Q.hid], h->data.data(), sizeof(float) * (size_t)H4 * Q.hid);
      for (int i = 0; i < H4; ++i) bih[(size_t)d * H4 + i] = b1->data[(size_t)i] + b2->data[(size_t)i];
    }
    Q.wih = (float*)dalloc(arena_, sizeof(float) * wih.size(), wih.data());
    Q.bih = (float*)dalloc(arena_, sizeof(float) * bih.size(), bih.data());
    Q.whh = (float*)dalloc(arena_, sizeof(float) * whh.size(), whh.data());
    if (!Q.wih || !Q.bih || !Q.whh) return false;
  }
  {
    const int K = 2 * Q.hid;
    const HostTensor *dw, *db;
    if (!need(lp + ".dense.0.weight", {Q.bins, K}, &dw) || !need(lp + ".dense.0.bias", {Q.bins}, &db) ||
        !fold_bn(lp + ".dense.1", Q.bins, db->data.data(), scale, shift))
      return false;
    const std::vector<float> sc(scale.begin(), scale.end()), sh(shift.begin(), shift.end());
    Q.wd = (float*)dalloc(arena_, sizeof(float) * dw->data.size(), dw->data.data());
    Q.dscale = (float*)dalloc(arena_, sizeof(float) * sc.size(), sc.data());
    Q.dshift = (float*)dalloc(arena_, sizeof(float) * sh.size(), sh.data());
    if (!Q.wd || !Q.dscale || !Q.dshift) return false;
  }
  Q.l0 = (float*)dalloc(arena_, sizeof(float) * (size_t)Nb * Q.T * Q.bins);
  Q.xp = (float*)dalloc(arena_, sizeof(float) * (size_t)Nb * Q.T * 8 * Q.hid);
  Q.hs = (float*)dalloc(arena_, sizeof(float) * (size_t)Nb * Q.T * 2 * Q.hid);
  Q.y = (float*)dalloc(arena_, sizeof(float) * (size_t)Nb * Q.T * Q.bins);
  return Q.l0 && Q.xp && Q.hs && Q.y;
}

bool Engine::finalize() {
  if (finalized_) return true;
  if (!err.empty() && !twiddle_) return false;
  const int max_bin = cfg_.n_fft / 2, W = cfg_.cropsize, Nb = cfg_.max_batch;
  const int nout = cfg_.nout, a1 = nout / 4, a2 = nout / 2;
  if (nout % 16) {
    err = "nout must be a multiple of 16";
    return false;
  }
  if (W - 2 * cfg_.offset <= 0) {   // lib/nets.py:129 assert
    err = "cropsize must be larger than 2*offset (AssertionError in the reference, lib/nets.py:129)";
    return false;
  }
  pos_aux2_ = 0; pos_aux1_ = a2; pos_x_ = a2 + a1;
  const int C3 = round_up(a2 + a1 + 2, 16);
  in3_ = make_buffer(arena_, Nb, max_bin, W, C3);
  o1_ = make_buffer(arena_, Nb, max_bin / 2, W, nout / 2);
  o2_ = make_buffer(arena_, Nb, max_bin / 2, W, nout);
  f3_ = make_buffer(arena_, Nb, max_bin, W, nout);
  if (!in3_.hi || !o1_.hi || !o2_.hi || !f3_.hi) return false;

  const int nin_lstm = max_bin / 2;
  // stage 1: input = [x]                      (lib/nets.py:59-65, 88-92)
  const int c0_1 = pos_x_ / 16 * 16, cp1 = round_up(pos_x_ + 2 - c0_1, 16);
  std::vector<int> p1((size_t)cp1, -1);
  p1[(size_t)(pos_x_ - c0_1)] = 0; p1[(size_t)(pos_x_ - c0_1 + 1)] = 1;
  // stage 2: input = cat[x, aux1]             (lib/nets.py:67-73, 95-98)
  const int c0_2 = pos_aux1_ / 16 * 16, cp2 = round_up(pos_x_ + 2 - c0_2, 16);
  std::vector<int> p2((size_t)cp2, -1);
  p2[(size_t)(pos_x_ - c0_2)] = 0; p2[(size_t)(pos_x_ - c0_2 + 1)] = 1;
  for (int j = 0; j < a1; ++j) p2[(size_t)(pos_aux1_ - c0_2 + j)] = 2 + j;
  // stage 3: input = cat[x, aux1, aux2]       (lib/nets.py:75-77, 101-102)
  std::vector<int> p3((size_t)C3, -1);
  p3[(size_t)pos_x_] = 0; p3[(size_t)pos_x_ + 1] = 1;
  for (int j = 0; j < a1; ++j) p3[(size_t)(pos_aux1_ + j)] = 2 + j;
  for (int j = 0; j < a2; ++j) p3[(size_t)(pos_aux2_ + j)] = 2 + a1 + j;

  const int Hb = max_bin / 2;
  if (!build_basenet(nets_[0], "stg1_low_band_net.0", p1, nout / 2, Hb, W, nin_lstm / 2, cfg_.nout_lstm) ||
      !build_basenet(nets_[1], "stg1_high_band_net", p1, nout / 4, Hb, W, nin_lstm / 2, cfg_.nout_lstm / 2) ||
      !build_basenet(nets_[2], "stg2_low_band_net.0", p2, nout, Hb, W, nin_lstm / 2, cfg_.nout_lstm) ||
      !build_basenet(nets_[3], "stg2_high_band_net", p2, nout / 2, Hb, W, nin_lstm / 2, cfg_.nout_lstm / 2) ||
      !build_basenet(nets_[4], "stg3_full_band_net", p3, nout, max_bin, W, nin_lstm, cfg_.nout_lstm))
    return false;
  if (!make_conv(bridge1_, "stg1_low_band_net.1", identity_perm(nout / 2, nout / 2), 1, 1, 1, 1, ACT_RELU, Hb, W) ||
      !make_conv(bridge2_, "stg2_low_band_net.1", identity_perm(nout, nout), 1, 1, 1, 1, ACT_RELU, Hb, W))
    return false;
  const HostTensor *ow, *aw;
  if (!need("out.weight", {2, nout, 1, 1}, &ow)) return false;
  if (!need("aux_out.weight", {2, 3 * nout / 4, 1, 1}, &aw)) return false;   // dead in forward, but a strict key
  out_w_ = (float*)dalloc(arena_, sizeof(float) * 2 * nout, ow->data.data());
  if (!out_w_) return false;
  // strict load: no unexpected keys (torch load_state_dict(strict=True), inference.py:131)
  {
    // every key outside the model's name space is unexpected
    for (auto& kv : sd_) {
      const std::string& k = kv.first;
      bool ok = k == "out.weight" || k == "aux_out.weight" || k.rfind("stg1_low_band_net.", 0) == 0 ||
                k.rfind("stg1_high_band_net.", 0) == 0 || k.rfind("stg2_low_band_net.", 0) == 0 ||
                k.rfind("stg2_high_band_net.", 0) == 0 || k.rfind("stg3_full_band_net.", 0) == 0;
      if (!ok) {
        err = "unexpected key in state_dict: " + k;
        return false;
      }
    }
  }
  if (!ck(cudaDeviceSynchronize(), "finalize")) return false;
  finalized_ = true;
  return true;
}

// ---------------------------------------------------------------------------------------------
void Engine::profile_enable(bool on) {
  for (auto& r : prof_) {
    cudaEventDestroy(r.a);
    cudaEventDestroy(r.b);
  }
  prof_.clear();
  profiling_ = on;
}

int Engine::prof_begin(const std::string& name, int kind, double flops, int N, int H, int W, cudaStream_t s) {
  if (!profiling_) return -1;
  ProfRec rec;
  cudaEventCreate(&rec.a);
  cudaEventCreate(&rec.b);
  rec.tc = kind; rec.flops = flops; rec.name = name;
  rec.N = N; rec.H = H; rec.W = W;
  cudaEventRecord(rec.a, s);
  prof_.push_back(rec);
  return (int)prof_.size() - 1;
}

void Engine::prof_end(int idx, cudaStream_t s) {
  if (idx >= 0) cudaEventRecord(prof_[(size_t)idx].b, s);
}

bool Engine::profile_read(double* out6) {
  for (int i = 0; i < 6; ++i) out6[i] = 0.0;
  for (auto& r : prof_) {
    if (r.tc > 1) continue;   // only the convolutions enter the roofline sums
    if (!ck(cudaEventSynchronize(r.b), "profile sync")) return false;
    float ms = 0.f;
    if (!ck(cudaEventElapsedTime(&ms, r.a, r.b), "profile elapsed")) return false;
    const int o = r.tc ? 0 : 3;
    out6[o] += ms;
    out6[o + 1] += r.flops;
    out6[o + 2] += 1.0;
  }
  return true;
}

bool Engine::profile_dump(std::string& text) {
  text.clear();
  char line[256];
  for (auto& r : prof_) {
    if (!ck(cudaEventSynchronize(r.b), "profile sync")) return false;
    float ms = 0.f;
    if (!ck(cudaEventElapsedTime(&ms, r.a, r.b), "profile elapsed")) return false;
    snprintf(line, sizeof(line), "%s %d %d %d %d %.6f %.6f\n", r.name.c_str(), r.N, r.H, r.W, r.tc, (double)ms,
             r.flops * 1e-9);
    text += line;
  }
  return true;
}

bool Engine::run_conv(const ConvLayer& L, const ActView& in, const ActView& out, cudaStream_t s, const ConvFusion& f) {
  const bool use_tc = L.tc != nullptr;
  if (!use_tc && !f.empty()) {
    err = "internal: fused work requested for a CUDA-core convolution";
    return false;
  }
  ++launches;
  if (!use_tc && cfg_.conv_mode == 0 && L.Cout >= 4 && !warned_simt_) {
    // loud, once per context: this geometry does not tile for the wgmma kernels (e.g. a cropsize whose feature-map
    // widths are not powers of two / multiples of 128) and runs on the fp32 CUDA-core kernel, an order of magnitude slower
    warned_simt_ = true;
    fprintf(stderr,
            "libvr_b200: WARNING: %s (N=%d, %dx%d -> %dx%d) does not tile for the tensor-core kernels and runs on the "
            "CUDA-core convolution; use a cropsize whose maps tile (e.g. 256) for full speed\n",
            L.name.c_str(), in.N, in.H, in.W, out.H, out.W);
  }
  // algorithmic FLOPs with the real (un-padded) channel counts: 2 * pixels * Cout * Cin * taps, over the computed
  // columns only (a fused output layer computes the kept ones)
  const int cols = f.mask ? out.W - 2 * f.mask->offset : out.W;
  const std::string name = L.name + (f.up ? "+up" : "") + (f.mask ? "+mask" : "");
  const int pi = prof_begin(name, use_tc ? 1 : 0, 2.0 * (double)out.N * out.H * cols * L.Cout * L.Cin * L.k * L.k,
                            out.N, out.H, out.W, s);
  bool ok;
  if (use_tc) {
    ok = ck(tc_launch(L, in, out, s, err, f), L.name.c_str());
  } else {
    ConvParams p;
    p.in = in; p.out = out;
    p.w = L.w; p.bias = L.bias;
    p.CinPad = L.CinPad; p.Cout = L.Cout; p.CoutPad = L.CoutPad;
    p.KH = L.k; p.KW = L.k; p.stride = L.stride;
    p.dil_h = L.dil_h; p.dil_w = L.dil_w;
    p.pad_h = L.dil_h * (L.k / 2); p.pad_w = L.dil_w * (L.k / 2);
    p.act = L.act;
    p.in.C = L.CinPad;
    g_last_conv = TcLastConv{};
    ok = ck(launch_conv_simt(p, s), L.name.c_str());
  }
  prof_end(pi, s);
  return ok;
}

bool Engine::run_decoder(const ConvLayer& L, const ActView& low, const Buffer& cat, int N, const ActView& out,
                         bool fused, cudaStream_t s, ConvFusion f) {
  if (fused) {
    f.up = &low;
    return run_conv(L, cat.all(N), out, s, f);
  }
  if (!timed("upsample2x", 1, N, cat.H, cat.W, s, [&] { return ck(launch_upsample2x(low, cat.view(N, 0, cat.H, 0, low.C), s), "decoder upsample"); }))
    return false;
  return run_conv(L, cat.all(N), out, s, f);
}

bool Engine::run_basenet(BaseNetPlan& P, const ActView& in, const ActView& out, int N, cudaStream_t s,
                         cudaStream_t side, const MaskOutParams* mask) {
  const int n = P.n, H = P.H;
  // encoders (lib/nets.py:27-31); each skip tensor is written straight into its decoder's concat buffer
  ActView e1 = P.cat1.view(N, 0, H, P.fused1 ? 0 : P.d2.C, n);   // staged: after up(h), which is as wide as d2
  if (!run_conv(P.enc1, in, e1, s)) return false;
  ActView e2 = P.cat2.view(N, 0, H / 2, P.fused2 ? 0 : 4 * n, 2 * n);
  if (!run_conv(P.enc_a[0], e1, P.t2.all(N), s) || !run_conv(P.enc_b[0], P.t2.all(N), e2, s)) return false;
  ActView e3 = P.cat3.view(N, 0, H / 4, 6 * n, 4 * n);
  if (!run_conv(P.enc_a[1], e2, P.t3.all(N), s) || !run_conv(P.enc_b[1], P.t3.all(N), e3, s)) return false;
  ActView e4 = P.cat4.view(N, 0, H / 8, 8 * n, 6 * n);
  if (!run_conv(P.enc_a[2], e3, P.t4.all(N), s) || !run_conv(P.enc_b[2], P.t4.all(N), e4, s)) return false;
  if (!run_conv(P.enc_a[3], e4, P.t5.all(N), s) || !run_conv(P.enc_b[3], P.t5.all(N), P.e5.all(N), s)) return false;
  // ASPP (lib/layers.py:92-105)
  const int c8 = 8 * n, h16 = H / 16;
  if (!timed("aspp.pool_freq_mean", 1, N, h16, P.W / 16, s, [&] { return ck(launch_pool_freq_mean(P.e5.all(N), P.pool.all(N), s), "aspp pool"); }))
    return false;
  if (!run_conv(P.aspp1, P.pool.all(N), P.f1.all(N), s)) return false;
  if (!timed("aspp.broadcast_rows", 1, N, h16, P.W / 16, s, [&] { return ck(launch_broadcast_rows(P.f1.all(N), P.acat.view(N, 0, h16, 0, c8), s), "aspp broadcast"); }))
    return false;
  if (!run_conv(P.aspp2, P.e5.all(N), P.acat.view(N, 0, h16, c8, c8), s)) return false;
  for (int i = 0; i < 3; ++i)
    if (!run_conv(P.aspp_d[i], P.e5.all(N), P.acat.view(N, 0, h16, (2 + i) * c8, c8), s)) return false;
  if (!run_conv(P.bott, P.acat.all(N), P.ao.all(N), s)) return false;
  // decoders (lib/nets.py:35-37, lib/layers.py:51-64)
  if (!timed("upsample2x", 1, N, H / 8, P.W / 8, s, [&] { return ck(launch_upsample2x(P.ao.all(N), P.cat4.view(N, 0, H / 8, 0, 8 * n), s), "up4"); }))
    return false;
  if (!run_conv(P.dec[0], P.cat4.all(N), P.d4.all(N), s)) return false;
  if (!timed("upsample2x", 1, N, H / 4, P.W / 4, s, [&] { return ck(launch_upsample2x(P.d4.all(N), P.cat3.view(N, 0, H / 4, 0, 6 * n), s), "up3"); }))
    return false;
  if (!run_conv(P.dec[1], P.cat3.all(N), P.d3.all(N), s)) return false;
  // The LSTM branch's 1x1 input convolution (2n -> 1, lib/layers.py:112,126) is one dot product per pixel of dec2's
  // output: the row kernel's epilogue accumulates it from the fp32 activations it is about to store.
  LstmPlan& Q = P.lstm;
  const ActView d2 = P.d2.all(N), h = P.d2.view(N, 0, H / 2, 0, 2 * n);
  ConvFusion dot;
  if (P.dot2) {
    if (!ck(cudaMemsetAsync(Q.l0, 0, sizeof(float) * (size_t)N * Q.bins * Q.T, s), "lstm conv clear")) return false;
    dot.dot_w = Q.conv_w;
    dot.dot_out = Q.l0;
  }
  if (!run_decoder(P.dec[2], P.d3.all(N), P.cat2, N, h, P.fused2, s, dot)) return false;
  // LSTM branch -> up(lstm), dec1's last reduction group (lib/nets.py:38, lib/layers.py:124-133).  Its 128-step
  // recurrence keeps only 2N CTAs busy, so when a side stream is free (stage 3) it runs there while the main stream
  // upsamples h for a staged dec1.
  const bool overlap = side != nullptr && !profiling_;
  cudaStream_t sl = overlap ? side : s;
  if (overlap) {
    if (!ck(cudaEventRecord(ev_lstm_fork_, s), "lstm fork") || !ck(cudaStreamWaitEvent(side, ev_lstm_fork_, 0), "lstm fork"))
      return false;
  }
  if (!P.dot2 &&
      !timed("lstm.inconv", 1, N, H / 2, P.W / 2, sl, [&] { return ck(launch_lstm_inconv(h, Q.conv_w, Q.l0, sl), "lstm conv"); }))
    return false;
  if (!timed("lstm.input_projection", 1, N, H / 2, P.W / 2, sl, [&] { return ck(launch_lstm_input_projection(Q.l0, Q.conv_bias, Q.wih, Q.bih, Q.xp, N, Q.T, Q.bins, 8 * Q.hid, sl), "lstm input projection"); }))
    return false;
  if (!timed("lstm.recurrence", 1, N, H / 2, P.W / 2, sl, [&] { return ck(launch_lstm_recurrence(Q.xp, Q.whh, Q.hs, N, Q.T, Q.hid, sl), "lstm recurrence"); }))
    return false;
  // the branch output at half resolution: fp32 plane y[bin][n][t]
  if (!timed("lstm.dense", 1, N, H / 2, P.W / 2, sl, [&] { return ck(launch_lstm_dense(Q.hs, Q.wd, Q.dscale, Q.dshift, N * Q.T, 2 * Q.hid, Q.bins, Q.y, sl), "lstm dense"); }))
    return false;
  const ActView up_lstm = P.lstm_own ? P.lstm_up.all(N) : P.cat1.view(N, 0, H, P.lstm_coff, 16);
  if (!timed("lstm.upsample2x", 1, N, H, P.W, sl, [&] { return ck(launch_upsample2x_c1(Q.y, Q.bins, Q.T, Q.T, (int64_t)N * Q.T, up_lstm, sl), "lstm upsample"); }))
    return false;
  // dec1 on cat[up(cat[h, lstm]), e1] (lib/nets.py:39): a fused dec1 produces up(d2) itself
  if (!P.fused1 &&
      !timed("upsample2x", 1, N, H, P.W, s, [&] { return ck(launch_upsample2x(h, P.cat1.view(N, 0, H, 0, 2 * n), s), "up1"); }))
    return false;
  if (overlap) {
    if (!ck(cudaEventRecord(ev_lstm_join_, side), "lstm join") || !ck(cudaStreamWaitEvent(s, ev_lstm_join_, 0), "lstm join"))
      return false;
  }
  ConvFusion f1;
  f1.up = P.fused1 ? &d2 : nullptr;
  f1.last_chunk = P.lstm_own ? &up_lstm : nullptr;
  f1.mask = mask;
  return run_conv(P.dec[3], P.cat1.all(N), out, s, f1);
}

bool Engine::forward(int N, const MaskOutParams& mask, cudaStream_t s) {
  const int max_bin = cfg_.n_fft / 2, Hb = max_bin / 2;
  const int nout = cfg_.nout, a1 = nout / 4, a2 = nout / 2;
  const int c0_1 = pos_x_ / 16 * 16, c0_2 = pos_aux1_ / 16 * 16;
  last_n_ = N;
  // Stages 1 and 2 (lib/nets.py:91-99): the low-band chain (stg1_low -> bridge -> stg2_low -> bridge) and the
  // high-band chain (stg1_high -> stg2_high) only meet at stage 3, so they run on two streams.
  const bool two = s_hi_ != nullptr && !profiling_;
  cudaStream_t sh = two ? s_hi_ : s;
  if (two) {
    if (!ck(cudaEventRecord(ev_fork_, s), "fork") || !ck(cudaStreamWaitEvent(s_hi_, ev_fork_, 0), "fork wait"))
      return false;
  }
  if (!run_basenet(nets_[1], in3_.view(N, Hb, Hb, c0_1, nets_[1].enc1.CinPad), in3_.view(N, Hb, Hb, pos_aux1_, a1), N,
                   sh))
    return false;
  if (!run_basenet(nets_[3], in3_.view(N, Hb, Hb, c0_2, nets_[3].enc1.CinPad), in3_.view(N, Hb, Hb, pos_aux2_, a2), N,
                   sh))
    return false;
  if (!run_basenet(nets_[0], in3_.view(N, 0, Hb, c0_1, nets_[0].enc1.CinPad), o1_.all(N), N, s)) return false;
  if (!run_conv(bridge1_, o1_.all(N), in3_.view(N, 0, Hb, pos_aux1_, a1), s)) return false;
  if (!run_basenet(nets_[2], in3_.view(N, 0, Hb, c0_2, nets_[2].enc1.CinPad), o2_.all(N), N, s)) return false;
  if (!run_conv(bridge2_, o2_.all(N), in3_.view(N, 0, Hb, pos_aux2_, a2), s)) return false;
  if (two) {
    if (!ck(cudaEventRecord(ev_join_, s_hi_), "join") || !ck(cudaStreamWaitEvent(s, ev_join_, 0), "join wait"))
      return false;
  }
  // Stage 3 (lib/nets.py:101-102) and the output layer (lib/nets.py:109-115, 127-129).  dec1 is a 3x3 convolution and
  // `out` a 1x1 one, so a kept frame needs dec1 at that frame only: where the row kernel can apply the output layer,
  // dec1 computes just the kept frames and writes the mask, and f3_ is not written.
  const ConvLayer& dec1 = nets_[4].dec[3];
  const bool crop = g_debug.crop_mask == 1 && dec1.tc && dec1.tc->fuses_mask(dec1.Cout, mask.offset, nets_[4].fused1);
  if (!run_basenet(nets_[4], in3_.all(N), f3_.all(N), N, s, two ? s_hi_ : nullptr, crop ? &mask : nullptr))
    return false;
  if (crop) return true;
  return timed("mask_out", 1, N, mask.f3.H, mask.f3.W, s, [&] { return ck(launch_mask_out(mask, s), "mask_out"); });
}

// ---------------------------------------------------------------------------------------------
bool Engine::predict_mask(const float* mag, int N, float* mask_out, int offset, cudaStream_t s) {
  const int max_bin = cfg_.n_fft / 2, nb = bins(), W = cfg_.cropsize, r = W - 2 * offset;
  for (int i = 0; i < N; i += cfg_.max_batch) {
    const int nb_now = N - i < cfg_.max_batch ? N - i : cfg_.max_batch;
    if (!timed("pack_mag_from_float", 1, nb_now, max_bin, W, s, [&] {
          return ck(launch_pack_mag_from_float(mag + (int64_t)i * 2 * nb * W, nb, max_bin, in3_.view(nb_now, 0, max_bin, pos_x_, 2), s), "pack");
        }))
      return false;
    MaskOutParams p;
    p.f3 = f3_.all(nb_now);
    p.w = out_w_;
    p.out = mask_out + (int64_t)i * 2 * nb * r;
    p.stride_n = (int64_t)2 * nb * r; p.stride_c = (int64_t)nb * r; p.stride_bin = r;
    p.offset = offset; p.t_base0 = 0; p.t_limit = r; p.roi_t = 0; p.accumulate = 0;
    if (!forward(nb_now, p, s)) return false;
  }
  return true;
}

bool Engine::separate_windows(const float2* spec, int64_t T, const float* norm, int pad_l, int first, int count,
                              float* mask, int64_t mask_T, int64_t frame_shift, int accumulate, cudaStream_t s,
                              bool final_pass) {
  const int max_bin = cfg_.n_fft / 2, nb = bins(), W = cfg_.cropsize, r = roi();
  for (int i = 0; i < count; i += cfg_.max_batch) {
    const int n_now = count - i < cfg_.max_batch ? count - i : cfg_.max_batch;
    const int g0 = first + i;
    if (!timed("pack_mag_from_spec", 1, n_now, max_bin, W, s, [&] {
          return ck(launch_pack_mag_from_spec(spec, nb, T, max_bin, W, r, pad_l, g0, norm, in3_.view(n_now, 0, max_bin, pos_x_, 2), s), "pack");
        }))
      return false;
    MaskOutParams p;
    p.f3 = f3_.all(n_now);
    p.w = out_w_;
    p.out = mask;
    p.stride_n = r; p.stride_c = (int64_t)nb * mask_T; p.stride_bin = mask_T;
    p.offset = cfg_.offset;
    p.t_base0 = (int64_t)g0 * r - frame_shift;
    p.t_limit = mask_T; p.roi_t = r; p.accumulate = accumulate;
    if (!forward(n_now, p, s)) return false;
    if (final_pass && on_frames_final_) {
      int64_t f = p.t_base0 + (int64_t)n_now * r;
      if (f > mask_T) f = mask_T;
      if (f > 0 && !on_frames_final_(f)) return false;
    }
  }
  return true;
}

bool Engine::normaliser(const float2* spec, int64_t T, int mode, float* out, cudaStream_t s) {
  const int64_t n = (int64_t)2 * bins() * T;
  if (mode == 0) return timed("normaliser.absmax", 1, 1, bins(), (int)T, s, [&] { return ck(launch_absmax(spec, n, out, s), "absmax"); });
  return timed("normaliser.lexmax", 2, 1, bins(), (int)T, s, [&] { return ck(launch_lexmax_abs(spec, n, ws_lex_, out, s), "lexmax"); });
}

// mask [2][bins][T]; the full window range of one track on this device (inference.py:70-77 / 83-98)
bool Engine::separate(const float2* spec, int64_t T, int tta, float* mask, cudaStream_t s) {
  const int r = roi();
  const int pad_l = cfg_.offset;
  // make_padding (lib/dataset.py:198-205): right = roi - (T % roi) + left
  const int64_t pad_r = r - (T % r) + pad_l;
  const int64_t Wpad = pad_l + T + pad_r;
  const int patches = (int)((Wpad - 2 * cfg_.offset) / r);
  if (!normaliser(spec, T, tta ? 1 : 0, ws_norm_, s)) return false;
  if (!separate_windows(spec, T, ws_norm_, pad_l, 0, patches, mask, T, 0, 0, s, !tta)) return false;
  if (tta) {
    const int64_t Wpad2 = Wpad + r;   // pad_l += roi/2, pad_r += roi/2 (inference.py:91-92)
    const int patches2 = (int)((Wpad2 - 2 * cfg_.offset) / r);
    if (!separate_windows(spec, T, ws_norm_, pad_l + r / 2, 0, patches2, mask, T, r / 2, 1, s, true)) return false;
  }
  return true;
}

bool Engine::apply_mask(const float2* spec, const float* mask, int64_t T, float2* y, float2* v, cudaStream_t s) {
  return timed("apply_mask", 1, 1, bins(), (int)T, s, [&] {
    return ck(launch_apply_mask(spec, mask, (int64_t)2 * bins() * T, y, v, s), "apply_mask");
  });
}

bool Engine::mask_frame_min(const float* mask, int64_t T, float* frame_min, cudaStream_t s) {
  return timed("mask_frame_min", 1, 1, bins(), (int)T, s, [&] {
    return ck(launch_mask_frame_min(mask, 2 * bins(), T, frame_min, s), "vr_mask_frame_min");
  });
}

bool Engine::mask_apply_weight(float* mask, int64_t T, const float* weight, cudaStream_t s) {
  return timed("mask_apply_weight", 1, 1, bins(), (int)T, s, [&] {
    return ck(launch_mask_apply_weight(mask, 2 * bins(), T, weight, s), "vr_mask_apply_weight");
  });
}

bool Engine::spec_image(const float2* spec, const float* mask, int64_t T, unsigned char* img_a, unsigned char* img_b,
                        cudaStream_t s) {
  if (T < 0 || !spec || !img_a || (mask && !img_b)) {
    err = "spec_image: needs spec, img_a, T >= 0 and, with a mask, img_b";
    return false;
  }
  // allocated on first use, once per context
  if (!ws_img_range_ && !(ws_img_range_ = (unsigned int*)dalloc(arena_, sizeof(unsigned int) * 4))) return false;
  return timed("spec_image", 2, 1, bins(), (int)T, s, [&] {
    return ck(launch_spec_image(spec, mask, (int64_t)bins() * T, ws_img_range_, img_a, img_b, s), "spec_image");
  });
}

bool Engine::vocal_image(const float2* spec_x, const float2* spec_y, int64_t T, unsigned char* img, cudaStream_t s) {
  if (T < 0 || !spec_x || !spec_y || !img) {
    err = "vocal_image: needs spec_x, spec_y, img and T >= 0";
    return false;
  }
  if (!ws_img_range_ && !(ws_img_range_ = (unsigned int*)dalloc(arena_, sizeof(unsigned int) * 4))) return false;
  return timed("vocal_image", 2, 1, bins(), (int)T, s, [&] {
    return ck(launch_vocal_image(spec_x, spec_y, (int64_t)bins() * T, ws_img_range_, img, s), "vocal_image");
  });
}

bool Engine::spec_sub(const float2* a, const float2* b, int64_t T, float2* out, cudaStream_t s) {
  if (T < 0 || !a || !b || !out) {
    err = "spec_sub: needs a, b, out and T >= 0";
    return false;
  }
  return timed("spec_sub", 1, 1, bins(), (int)T, s, [&] {
    return ck(launch_spec_sub(a, b, (int64_t)2 * bins() * T, out, s), "spec_sub");
  });
}

bool Engine::oracle_mask(const float2* spec_x, const float2* spec_y, int64_t T, int kind, float* mask, cudaStream_t s) {
  if (T < 1 || kind < 0 || kind > 3 || !spec_x || !spec_y || !mask) {
    err = "oracle_mask: needs spec_x, spec_y, mask, T >= 1 and kind 0 (iam), 1 (ibm), 2 (irm1) or 3 (irm2)";
    return false;
  }
  return timed("oracle_mask", 1, 1, bins(), (int)T, s, [&] {
    return ck(launch_oracle_mask(spec_x, spec_y, (int64_t)2 * bins() * T, kind, mask, s), "oracle_mask");
  });
}

// train.py:108-134 validate_epoch over lib/dataset.py:220-248 make_validation_set, one pair: coef = max(max|X|, max|y|),
// ceil(T / roi) windows of X / coef padded by make_padding (left = offset) through the net, then the L1 sums of the
// kept mask frames.  Only the mask workspace is needed (no inverse STFT, so not ensure_ws's frame workspace).
bool Engine::validation_loss(const float2* spec_x, const float2* spec_y, int64_t T, float* coef_out,
                             double* window_sums, cudaStream_t s) {
  if (T < 1 || !spec_x || !spec_y || !window_sums) {
    err = "validation_loss: needs spec_x, spec_y, window_sums and T >= 1";
    return false;
  }
  if (cfg_.cropsize <= 2 * cfg_.offset) {
    err = "validation_loss: cropsize must exceed 2 * offset (the reference's predict keeps no frame otherwise)";
    return false;
  }
  const int r = roi();
  const int64_t n64 = (T + r - 1) / r;   // lib/dataset.py:236, not Separator's (W_pad - 2*offset) // roi
  if (n64 > (int64_t)INT32_MAX / 2) {
    err = "validation_loss: track too long";
    return false;
  }
  const int n = (int)n64;
  const int64_t mask_T = n64 * r;
  const int64_t nmask = (int64_t)2 * bins() * mask_T;
  if (!ck(ws_mask_.ensure(nmask), "workspace mask") ||
      !ck(ws_val_.ensure(validation_l1_scratch(n)), "workspace validation"))
    return false;
  float* coef = coef_out ? coef_out : ws_norm_;
  const int64_t nspec = (int64_t)2 * bins() * T;
  if (!timed("normaliser.absmax", 2, 1, bins(), (int)T, s, [&] {
        return ck(launch_absmax(spec_x, nspec, coef, s), "absmax X") &&
               ck(launch_absmax(spec_y, nspec, coef, s, true), "absmax y");
      }))
    return false;
  if (!separate_windows(spec_x, T, coef, cfg_.offset, 0, n, ws_mask_.get(), mask_T, 0, 0, s)) return false;
  return timed("validation_l1", 2, n, bins(), r, s, [&] {
    return ck(launch_validation_l1(spec_x, spec_y, ws_mask_.get(), bins(), T, r, n, coef, ws_val_.get(), window_sums, s),
              "validation_l1");
  });
}

bool Engine::wiener(const float2* spec, float2* y, float2* v, int64_t T, int iterations, cudaStream_t s) {
  if (T < 1 || iterations < 0 || !spec || !y || !v) {
    err = "wiener: needs spec, y_spec, v_spec, T >= 1 and iterations >= 0";
    return false;
  }
  if (iterations == 0) return true;
  if (!ck(ws_wiener_.ensure(wiener_scratch(bins())), "workspace wiener")) return false;
  return timed("wiener", 1 + 3 * iterations, 1, bins(), (int)T, s, [&] {
    return ck(launch_wiener(spec, y, v, bins(), T, iterations, ws_wiener_.get(), s), "wiener");
  });
}

bool Engine::stft(const float* wave, int64_t L, float2* spec, int64_t T, float* absmax, cudaStream_t s) {
  if (!stft_range(wave, L, spec, T, 0, T, s)) return false;
  if (absmax) return normaliser(spec, T, 0, absmax, s);
  return true;
}

// frames [t0, t1) of the track only: what a rank of the window-sharded path needs (lib/distributed.py)
bool Engine::stft_range(const float* wave, int64_t L, float2* spec, int64_t T, int64_t t0, int64_t t1, cudaStream_t s) {
  if (T != 1 + L / cfg_.hop) {
    err = "stft: T must equal 1 + L // hop_length";
    return false;
  }
  if (t0 < 0 || t1 > T || t0 > t1) {
    err = "stft: frame range outside [0, T]";
    return false;
  }
  return timed("stft", 1, 1, bins(), (int)(t1 - t0), s, [&] { return ck(launch_stft(wave, L, cfg_.n_fft, cfg_.hop, spec, T, t0, t1, twiddle_, window_, s), "stft"); });
}

bool Engine::normaliser_range(const float2* spec, int64_t T, int64_t t0, int64_t t1, float* out, cudaStream_t s) {
  if (t0 < 0 || t1 > T || t0 > t1) {
    err = "normaliser: frame range outside [0, T]";
    return false;
  }
  return timed("normaliser.absmax_range", 1, 1, bins(), (int)(t1 - t0), s, [&] {
    return ck(launch_absmax_range(spec, 2 * bins(), T, t0, t1, out, s), "absmax range");
  });
}

bool Engine::ensure_ws(int64_t T) {
  const int64_t nspec = (int64_t)2 * bins() * T;
  return ck(ws_spec_.ensure(nspec), "workspace spec") && ck(ws_mask_.ensure(nspec), "workspace mask") &&
         ck(ws_frames_.ensure((int64_t)4 * T * cfg_.n_fft), "workspace frames");
}

bool Engine::istft(const float2* spec, const float* mask, int64_t T, float* wave_a, float* wave_b, cudaStream_t s) {
  return istft_range(spec, mask, T, 0, T - 1, wave_a, wave_b, s);
}

// Frames past its own index that output hop k reads: its last sample, hop*k + hop - 1, lies at hop*k + hop - 1 + NF/2
// in the centre-padded signal, and the last window reaching that is frame k + ceil(NF / (2*hop)).
int64_t Engine::istft_lookahead() const { return (cfg_.n_fft / 2 + cfg_.hop - 1) / cfg_.hop; }

// Output hops [k0, k1) (samples [hop*k0, hop*k1)) of wave [2][hop*(T-1)]; reads frames of spec / mask that overlap
// them (k0 + 1 - istft_lookahead() .. k1 - 1 + istft_lookahead() clipped to the track; k0..k1 for hop = n_fft/2).
// wave_a / wave_b may point into another GPU's memory (peer-mapped).
bool Engine::istft_range(const float2* spec, const float* mask, int64_t T, int64_t k0, int64_t k1, float* wave_a,
                         float* wave_b, cudaStream_t s) {
  if (k0 < 0 || k1 > T - 1 || k0 > k1) {
    err = "istft: hop range outside [0, T-1]";
    return false;
  }
  if (k1 == k0) return true;
  const int NF = cfg_.n_fft, hop = cfg_.hop;
  // first frame touching samples [hop*k0, hop*k1): u = s + NF/2, frames ceil((u-NF+1)/hop) .. floor(u/hop)
  int64_t f0 = ((int64_t)hop * k0 + NF / 2 - NF + hop) / hop;
  if ((int64_t)hop * k0 + NF / 2 - NF + 1 <= 0) f0 = 0;
  int64_t f1 = k1 - 1 + istft_lookahead();
  if (f1 > T - 1) f1 = T - 1;
  const int64_t nfr = f1 - f0 + 1;
  if (!ck(ws_frames_.ensure((int64_t)4 * nfr * NF), "workspace frames")) return false;
  float* fa = ws_frames_.get();
  float* fb = mask ? fa + (int64_t)2 * nfr * NF : nullptr;
  if (!timed("istft.frames", 1, 1, bins(), (int)nfr, s, [&] { return ck(launch_istft_frames(spec, mask, NF, T, f0, nfr, fa, fb, twiddle_, window_, s), "istft frames"); }))
    return false;
  return timed("istft.overlap_add", 1, 1, bins(), (int)nfr, s, [&] {
    return ck(launch_istft_ola(fa, fb, NF, hop, T, f0, nfr, (int64_t)hop * k0, (int64_t)hop * k1, wave_a, mask ? wave_b : nullptr, window_, s), "istft ola");
  });
}

// wave (2, L) in HBM -> instruments / vocals waves (2, hop*(T-1)) in HBM: the whole inference.py:147-176 path.
bool Engine::separate_wave(const float* wave, int64_t L, int tta, float* inst, float* voc, cudaStream_t s) {
  const int64_t T = 1 + L / cfg_.hop;
  if (!ensure_ws(T)) return false;
  if (!stft(wave, L, ws_spec_.get(), T, nullptr, s)) return false;
  if (!separate(ws_spec_.get(), T, tta, ws_mask_.get(), s)) return false;
  return istft(ws_spec_.get(), ws_mask_.get(), T, inst, voc, s);
}

// Host-buffer entry (the end-to-end call): H2D of the wave, the whole path, D2H of both stems.
bool Engine::separate_wave_host(const float* wave, int64_t L, int tta, float* inst, float* voc, cudaStream_t s,
                                unsigned char* img_inst, unsigned char* img_voc) {
  const int64_t T = 1 + L / cfg_.hop;
  const int64_t Lo = (int64_t)cfg_.hop * (T - 1);
  if (!ck(ws_wave_.ensure(2 * L + 4 * Lo), "workspace wave")) return false;
  const int64_t img_bytes = (int64_t)3 * bins() * T;
  if ((img_inst || img_voc) && !ck(ws_img_.ensure(2 * img_bytes), "workspace images")) return false;
  float* d_in = ws_wave_.get();
  float* d_inst = d_in + 2 * L;
  float* d_voc = d_inst + 2 * Lo;
  if (!ck(cudaMemcpyAsync(d_in, wave, sizeof(float) * 2 * L, cudaMemcpyHostToDevice, s), "H2D wave")) return false;
  // The stems leave the device span by span: as soon as a window batch of the last pass has written its mask frames,
  // the masked inverse STFT of the hops they complete runs on `s` and their device-to-host copy on the copy stream,
  // overlapped with the next batch of the net (the copies of a 4-minute track are 169 MB).
  if (!ensure_ws(T)) return false;
  float2* spec = ws_spec_.get();
  float* mask = ws_mask_.get();
  if (!stft(d_in, L, spec, T, nullptr, s)) return false;
  int64_t k_done = 0;
  bool ok = true;
  auto flush = [&](int64_t f) -> bool {
    // mask frames [0, f) are final: output hop k is finished once k + istft_lookahead() < f (k + 1 < f for
    // hop = n_fft/2); frames from f on may still hold the previous track's mask, or only the first pass of --tta
    int64_t k1 = f >= T ? T - 1 : f - istft_lookahead();
    if (k1 <= k_done) return true;
    if (!istft_range(spec, mask, T, k_done, k1, d_inst, d_voc, s)) return false;
    if (!ck(cudaEventRecord(ev_span_, s), "span event") || !ck(cudaStreamWaitEvent(s_copy_, ev_span_, 0), "span wait"))
      return false;
    const size_t off = (size_t)cfg_.hop * (size_t)k_done, cnt = (size_t)cfg_.hop * (size_t)(k1 - k_done);
    for (int c = 0; c < 2; ++c) {
      if (!ck(cudaMemcpyAsync(inst + (size_t)c * Lo + off, d_inst + (size_t)c * Lo + off, sizeof(float) * cnt,
                              cudaMemcpyDeviceToHost, s_copy_), "D2H inst") ||
          !ck(cudaMemcpyAsync(voc + (size_t)c * Lo + off, d_voc + (size_t)c * Lo + off, sizeof(float) * cnt,
                              cudaMemcpyDeviceToHost, s_copy_), "D2H voc"))
        return false;
    }
    k_done = k1;
    return true;
  };
  on_frames_final_ = flush;
  ok = separate(spec, T, tta, mask, s);
  on_frames_final_ = nullptr;
  if (ok) ok = flush(T);
  if (ok && (img_inst || img_voc)) {
    // after the last span: the images of the final mask, copied back behind the stems on the copy stream
    unsigned char* img = ws_img_.get();
    ok = spec_image(spec, mask, T, img, img + img_bytes, s) &&
         ck(cudaEventRecord(ev_span_, s), "image event") && ck(cudaStreamWaitEvent(s_copy_, ev_span_, 0), "image wait") &&
         (!img_inst || ck(cudaMemcpyAsync(img_inst, img, img_bytes, cudaMemcpyDeviceToHost, s_copy_), "D2H image")) &&
         (!img_voc || ck(cudaMemcpyAsync(img_voc, img + img_bytes, img_bytes, cudaMemcpyDeviceToHost, s_copy_),
                         "D2H image"));
  }
  if (!ok) {
    cudaStreamSynchronize(s);
    cudaStreamSynchronize(s_copy_);
    return false;
  }
  return ck(cudaStreamSynchronize(s), "separate_wave_host sync") && ck(cudaStreamSynchronize(s_copy_), "separate_wave_host copy sync");
}

// ---------------------------------------------------------------------------------------------
bool Engine::debug_weights(ConvLayer& L, Arena& arena, const float* w, const float* bias, int Cout, int Cin,
                           const std::vector<int>& perm, bool use_tc, int H, int W, bool rows_wide, cudaStream_t s) {
  std::vector<float> hw((size_t)Cout * Cin * L.k * L.k), hb((size_t)Cout);
  if (!ck(cudaMemcpyAsync(hw.data(), w, hw.size() * sizeof(float), cudaMemcpyDeviceToHost, s), "weights to host") ||
      !ck(cudaMemcpyAsync(hb.data(), bias, hb.size() * sizeof(float), cudaMemcpyDeviceToHost, s), "bias to host") ||
      !ck(cudaStreamSynchronize(s), "weights to host"))
    return false;
  const std::vector<double> one((size_t)Cout, 1.0), shift(hb.begin(), hb.end());
  std::vector<float> wp, bp;
  pack_conv(L, hw.data(), Cout, Cin, one.data(), shift.data(), perm, wp, bp);
  return prepare_conv(L, arena, wp, bp, use_tc, H, W, rows_wide);
}

bool Engine::to_nchw(const ActView& v, int C, float* y_nchw, cudaStream_t s) {
  return timed("act_to_nchw", 1, v.N, v.H, v.W, s,
               [&] { return ck(launch_act_to_nchw(v, C, y_nchw, s), "act_to_nchw"); });
}

bool Engine::debug_conv(const float* x_nchw, int N, int Cin, int H, int W, const float* w, const float* bias, int Cout,
                        int k, int stride, int dil_h, int dil_w, int act, int use_tc, float* y_nchw, cudaStream_t s) {
  const int cin_pad = round_up(Cin, 16);
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  Arena arena;   // the hook's buffers and weights, freed on return
  const Buffer bin = make_buffer(arena, N, H, W, cin_pad);
  const Buffer bout = make_buffer(arena, N, Ho, Wo, round_up(Cout, 8));
  ConvLayer L;
  L.name = "debug_conv";
  L.k = k; L.stride = stride; L.dil_h = dil_h; L.dil_w = dil_w; L.act = act;
  // vr_debug_set(2, 1): exercise the 64-wide row tile on a plain convolution
  if (!bin.hi || !bout.hi ||
      !debug_weights(L, arena, w, bias, Cout, Cin, identity_perm(Cin, cin_pad), use_tc != 0, Ho, Wo,
                     g_debug.rows_wide == 1, s))
    return false;
  if (use_tc && !L.tc) {
    err = "debug_conv: geometry not supported by the wgmma kernel";
    return false;
  }
  if (!timed("nchw_to_act", 1, N, H, W, s,
             [&] { return ck(launch_nchw_to_act(x_nchw, Cin, bin.all(N), s), "nchw_to_act"); }))
    return false;
  const ActView out = bout.view(N, 0, Ho, 0, Cout);
  const int saved_mode = cfg_.conv_mode;
  cfg_.conv_mode = use_tc ? 0 : 1;   // a requested CUDA-core run is not warned about
  const bool ok = run_conv(L, bin.all(N), out, s);
  cfg_.conv_mode = saved_mode;
  return ok && to_nchw(out, Cout, y_nchw, s) && ck(cudaStreamSynchronize(s), "debug_conv sync");
}

// Test hook for the decoder path: y = act(conv3x3(cat[up2x(low), skip]) + bias), fused (upsample inside the row
// kernel) or staged (upsample kernel, then convolution), with the concat buffer laid out as the engine's decoders'.
bool Engine::debug_decoder(const float* low_nchw, int N, int Cl, int h, int w, const float* skip_nchw, int Cs,
                           const float* wgt, const float* bias, int Cout, int act, int fused, float* y_nchw,
                           cudaStream_t s) {
  const int H = 2 * h, W = 2 * w;
  const int cl_pad = round_up(Cl, 32), cin_pad = round_up(cl_pad + Cs, 16);
  const int skip_off = fused ? 0 : cl_pad;   // the fused kernel's concat buffer holds only the skip channels
  Arena arena;   // the hook's buffers and weights, freed on return
  const Buffer blow = make_buffer(arena, N, h, w, cl_pad);
  const Buffer bcat = make_buffer(arena, N, H, W, cin_pad - cl_pad + skip_off);
  const Buffer bout = make_buffer(arena, N, H, W, round_up(Cout, 16));
  ConvLayer L;
  L.name = "debug_decoder";
  L.k = 3; L.act = act;
  std::vector<int> perm((size_t)cin_pad, -1);   // reduction order: [up Cl | pad | skip Cs]
  for (int i = 0; i < Cl; ++i) perm[(size_t)i] = i;
  for (int i = 0; i < Cs; ++i) perm[(size_t)(cl_pad + i)] = Cl + i;
  if (!blow.hi || !bcat.hi || !bout.hi ||
      !debug_weights(L, arena, wgt, bias, Cout, Cl + Cs, perm, true, H, W, true, s))
    return false;
  if (fused && !(L.tc && L.tc->fuses_upsample(blow.C))) {
    err = "debug_decoder: geometry not supported by the fused row kernel";
    return false;
  }
  const ActView skip = bcat.view(N, 0, H, skip_off, cin_pad - cl_pad);
  if (!timed("nchw_to_act", 1, N, h, w, s,
             [&] { return ck(launch_nchw_to_act(low_nchw, Cl, blow.all(N), s), "nchw_to_act low"); }) ||
      !timed("nchw_to_act", 1, N, H, W, s,
             [&] { return ck(launch_nchw_to_act(skip_nchw, Cs, skip, s), "nchw_to_act skip"); }))
    return false;
  const ActView out = bout.view(N, 0, H, 0, Cout);
  return run_decoder(L, blow.all(N), bcat, N, out, fused != 0, s) && to_nchw(out, Cout, y_nchw, s) &&
         ck(cudaStreamSynchronize(s), "debug_decoder sync");
}

// Every activation buffer and LSTM plane is an allocation of its own (build_basenet, finalize), so after a forward each
// one still holds what that forward wrote into it.
bool Engine::debug_tensor(const std::string& name, int n0, int n, float* out, int64_t* shape4, cudaStream_t s) {
  if (n0 < 0 || n < 0 || n0 + n > cfg_.max_batch) {
    err = "debug_tensor: images [" + std::to_string(n0) + ", " + std::to_string(n0 + n) + ") outside [0, max_batch = " +
          std::to_string(cfg_.max_batch) + ")";
    return false;
  }
  const Buffer* buf = name == "in3" ? &in3_ : name == "o1" ? &o1_ : name == "o2" ? &o2_ : name == "f3" ? &f3_ : nullptr;
  const BaseNetPlan* P = nullptr;
  std::string member;
  for (const BaseNetPlan& q : nets_)
    if (name.size() > q.prefix.size() + 1 && name.compare(0, q.prefix.size() + 1, q.prefix + ".") == 0) {
      P = &q;
      member = name.substr(q.prefix.size() + 1);
    }
  if (P) {
    const std::pair<const char*, const Buffer*> members[] = {
        {"cat1", &P->cat1}, {"lstm_up", &P->lstm_up}, {"t2", &P->t2}, {"cat2", &P->cat2}, {"t3", &P->t3},
        {"cat3", &P->cat3}, {"t4", &P->t4}, {"cat4", &P->cat4}, {"t5", &P->t5}, {"e5", &P->e5}, {"pool", &P->pool},
        {"f1", &P->f1}, {"acat", &P->acat}, {"ao", &P->ao}, {"d4", &P->d4}, {"d3", &P->d3}, {"d2", &P->d2}};
    for (const auto& m : members)
      if (member == m.first) buf = m.second;
    if (member == "lstm_up" && !P->lstm_own) {
      err = "debug_tensor: " + P->prefix + " has no lstm_up buffer (its up(lstm) group is a channel slice of cat1)";
      return false;
    }
  }
  if (buf) {
    const int64_t shape[4] = {n, buf->C, buf->H, buf->W};
    for (int i = 0; i < 4; ++i) shape4[i] = shape[i];
    if (!out) return true;
    ActView v = buf->all(n);
    v.hi += (int64_t)n0 * v.sn;
    v.lo += (int64_t)n0 * v.sn;
    return to_nchw(v, buf->C, out, s);
  }
  // LSTM planes in logical layouts: l0 / y (n, bins, T), xp (n, T, 8 hid), hs (n, T, 2 hid); shape4[3] = 1
  const LstmPlan* Q = P ? &P->lstm : nullptr;
  const float* src = nullptr;
  int64_t d1 = 0, d2 = 0;
  if (Q && member == "lstm.l0") { src = Q->l0; d1 = Q->bins; d2 = Q->T; }
  if (Q && member == "lstm.xp") { src = Q->xp; d1 = Q->T; d2 = 8 * Q->hid; }
  if (Q && member == "lstm.hs") { src = Q->hs; d1 = Q->T; d2 = 2 * Q->hid; }
  if (Q && member == "lstm.y") { src = Q->y; d1 = Q->bins; d2 = Q->T; }
  if (!src) {
    err = "debug_tensor: unknown tensor name " + name;
    return false;
  }
  const int64_t shape[4] = {n, d1, d2, 1};
  for (int i = 0; i < 4; ++i) shape4[i] = shape[i];
  if (!out) return true;
  if (member != "lstm.y")
    return ck(cudaMemcpyAsync(out, src + (int64_t)n0 * d1 * d2, sizeof(float) * (size_t)(n * d1 * d2),
                              cudaMemcpyDeviceToDevice, s), "debug_tensor copy");
  // y is stored [bin][image][t] with the last forward's batch as the image count
  if (n0 + n > last_n_) {
    err = "debug_tensor: the last forward ran " + std::to_string(last_n_) + " images; " + name + " has no image " +
          std::to_string(n0 + n - 1);
    return false;
  }
  for (int i = 0; i < n; ++i)
    if (!ck(cudaMemcpy2DAsync(out + (int64_t)i * d1 * d2, sizeof(float) * (size_t)d2,
                              src + (int64_t)(n0 + i) * d2, sizeof(float) * (size_t)last_n_ * d2,
                              sizeof(float) * (size_t)d2, (size_t)d1, cudaMemcpyDeviceToDevice, s),
            "debug_tensor copy"))
      return false;
  return true;
}

}  // namespace vr
