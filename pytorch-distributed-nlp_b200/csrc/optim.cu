// Gradient exchange + optimizer in one pass over HBM.
//
// Replaces three things the reference does separately and un-overlapped (SURVEY.md K13-K15):
//   optimizer.zero_grad()            multi-gpu-distributed-cls.py:172   (grads are consumed in place, never re-zeroed)
//   DDP Reducer bucket all-reduce    SP/torch/nn/parallel/distributed.py:1255-1280, reducer.hpp:276-286
//   HF AdamW.step python loop        transformers 4.28.1 optimization.py::AdamW.step (~1600 launches/step)
//
// Each rank owns a contiguous 1/world slice of every bucket: it reads that slice of the bf16 gradients straight
// out of every peer's HBM (NVSwitch peer loads), sums in fp32 in fixed rank order, divides by world (DDP's mean),
// applies the optimizer update (HF AdamW, or torch SGD) to its fp32 master weights / state, and stores the refreshed
// bf16 shadow weights into every peer's weight buffer (NVSwitch peer stores).  world == 1 degenerates to a fused
// multi-tensor optimizer step.
#include "common.cuh"
#include "../../include/b2_ddp_bert.h"

namespace b2 {

constexpr int MAX_WORLD = 8;

// ---- update rules --------------------------------------------------------------------------------------------------
// The two kernel forms below (reduce_update_kernel: any world; slim_update_kernel: world 1, beside the backward) own the
// gradient path every optimizer shares: the peer gather in rank order, 1/world and the GradScaler unscale, the clip
// coefficient, the fp32 stash, the found_inf skip, the device lr and the delivery of the bf16 shadow weights.  They are
// instantiated once per update rule.  A rule supplies
//   Args                            its scalars (pre-rounded on the host) and state pointers
//   Step reduce_step / slim_step    the per-launch values, from the device lr when lr_dev is set
//   update8 (reduce form)           8 elements: loads master + state, updates, stores them, returns the new weights
//   update4 (slim form)             4 elements, the same
struct AdamWRule {
  struct Args {
    float* m; float* v;
    // scalars pre-rounded on the host exactly as torch rounds the python doubles HF AdamW passes to its ATen ops
    double lr_d, beta1_d, beta2_d, weight_decay_d;
    float lr, beta1, beta2, one_minus_beta1, one_minus_beta2, eps, lr_wd;
    int correct_bias;
    const long long* step_counter;   // reduce form: t = *step_counter + 1
    const float* step_size;          // slim form: the bias-corrected step size from adamw_prepare_kernel
  };
  struct Step { float step_size, lr_wd; };

  static __device__ __forceinline__ Step reduce_step(const Args& a, const double* lr_dev) {
    // the learning rate from device memory: the same double arithmetic the host does on the by-value lr, so a device
    // lr equal to the host value gives the same bits
    double lr_d = a.lr_d;
    float lr = a.lr, lr_wd = a.lr_wd;
    if (lr_dev != nullptr) {
      lr_d = *lr_dev;
      lr = (float)lr_d;
      lr_wd = (float)(lr_d * a.weight_decay_d);
    }
    // HF AdamW bias correction: step_size = lr * sqrt(1 - b2^t) / (1 - b1^t), t = steps taken including this one
    const long long t = *a.step_counter + 1;
    float step_size = lr;
    if (a.correct_bias) {
      const double bc1 = 1.0 - pow(a.beta1_d, (double)t);
      const double bc2 = 1.0 - pow(a.beta2_d, (double)t);
      step_size = (float)(lr_d * sqrt(bc2) / bc1);
    }
    return {step_size, lr_wd};
  }
  static __device__ __forceinline__ Step slim_step(const Args& a, const double* lr_dev) {
    return {*a.step_size, lr_dev != nullptr ? (float)(*lr_dev * a.weight_decay_d) : a.lr_wd};
  }

  template <class P>
  static __device__ __forceinline__ void update8(const P& p, const Step& s, long long e, const float* g,
                                                 float inv_world, float coef, bool decay, float* w) {
    const Args& a = p.rule;
    float4 w0 = *reinterpret_cast<const float4*>(p.master + e), w1 = *reinterpret_cast<const float4*>(p.master + e + 4);
    float4 m0 = *reinterpret_cast<const float4*>(a.m + e), m1 = *reinterpret_cast<const float4*>(a.m + e + 4);
    float4 v0 = *reinterpret_cast<const float4*>(a.v + e), v1 = *reinterpret_cast<const float4*>(a.v + e + 4);
    w[0] = w0.x; w[1] = w0.y; w[2] = w0.z; w[3] = w0.w; w[4] = w1.x; w[5] = w1.y; w[6] = w1.z; w[7] = w1.w;
    float mm[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
    float vv[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float gk = g[k] * inv_world * coef;
      mm[k] = mm[k] * a.beta1 + gk * a.one_minus_beta1;
      vv[k] = vv[k] * a.beta2 + gk * gk * a.one_minus_beta2;
      const float denom = sqrtf(vv[k]) + a.eps;
      w[k] = w[k] - s.step_size * (mm[k] / denom);
      if (decay) w[k] = w[k] - s.lr_wd * w[k];
    }
    *reinterpret_cast<float4*>(p.master + e) = make_float4(w[0], w[1], w[2], w[3]);
    *reinterpret_cast<float4*>(p.master + e + 4) = make_float4(w[4], w[5], w[6], w[7]);
    *reinterpret_cast<float4*>(a.m + e) = make_float4(mm[0], mm[1], mm[2], mm[3]);
    *reinterpret_cast<float4*>(a.m + e + 4) = make_float4(mm[4], mm[5], mm[6], mm[7]);
    *reinterpret_cast<float4*>(a.v + e) = make_float4(vv[0], vv[1], vv[2], vv[3]);
    *reinterpret_cast<float4*>(a.v + e + 4) = make_float4(vv[4], vv[5], vv[6], vv[7]);
  }

  template <class P>
  static __device__ __forceinline__ float4 update4(const P& p, const Step& s, long long e, uint2 q, float coef) {
    const Args& a = p.rule;
    float4 mm = *reinterpret_cast<const float4*>(a.m + e);
    float4 vv = *reinterpret_cast<const float4*>(a.v + e);
    const float g0 = bf16_lo(q.x) * coef, g1 = bf16_hi(q.x) * coef, g2 = bf16_lo(q.y) * coef,
                g3 = bf16_hi(q.y) * coef;
    mm.x = mm.x * a.beta1 + g0 * a.one_minus_beta1; vv.x = vv.x * a.beta2 + g0 * g0 * a.one_minus_beta2;
    mm.y = mm.y * a.beta1 + g1 * a.one_minus_beta1; vv.y = vv.y * a.beta2 + g1 * g1 * a.one_minus_beta2;
    mm.z = mm.z * a.beta1 + g2 * a.one_minus_beta1; vv.z = vv.z * a.beta2 + g2 * g2 * a.one_minus_beta2;
    mm.w = mm.w * a.beta1 + g3 * a.one_minus_beta1; vv.w = vv.w * a.beta2 + g3 * g3 * a.one_minus_beta2;
    *reinterpret_cast<float4*>(a.m + e) = mm;
    *reinterpret_cast<float4*>(a.v + e) = vv;
    // the Adam direction first, then the master weights: fewer values live at once (no spills at 32 registers)
    float4 u;
    u.x = mm.x / (sqrtf(vv.x) + a.eps);
    u.y = mm.y / (sqrtf(vv.y) + a.eps);
    u.z = mm.z / (sqrtf(vv.z) + a.eps);
    u.w = mm.w / (sqrtf(vv.w) + a.eps);
    float4 w = *reinterpret_cast<const float4*>(p.master + e);
    const bool decay = p.has_wd && p.decay[e >> 3];
    w.x = w.x - s.step_size * u.x;
    w.y = w.y - s.step_size * u.y;
    w.z = w.z - s.step_size * u.z;
    w.w = w.w - s.step_size * u.w;
    if (decay) {
      w.x = w.x - s.lr_wd * w.x; w.y = w.y - s.lr_wd * w.y; w.z = w.z - s.lr_wd * w.z; w.w = w.w - s.lr_wd * w.w;
    }
    *reinterpret_cast<float4*>(p.master + e) = w;
    return w;
  }
};

// torch.optim.SGD (torch 2.11 sgd.py::_single_tensor_sgd), per element.  Each `x.add(y, alpha=a)` of torch's CUDA ops
// is one fma(a, y, x) and `buf.mul_(momentum)` a separately rounded product, so those are written out explicitly.
struct SgdRule {
  struct Args {
    float* buf;                      // momentum buffer; NULL when momentum == 0 (then never read or written)
    const long long* step_counter;   // applied steps since the buffer exists: 0 = torch's `momentum_buffer is None`
    float neg_lr, momentum, one_minus_dampening, weight_decay;   // -lr, 1 - dampening: rounded as torch's alphas
    int nesterov, maximize;
  };
  struct Step { float neg_lr; bool first; };

  static __device__ __forceinline__ Step reduce_step(const Args& a, const double* lr_dev) {
    return {lr_dev != nullptr ? (float)(-*lr_dev) : a.neg_lr, a.buf != nullptr && *a.step_counter == 0};
  }
  static __device__ __forceinline__ Step slim_step(const Args& a, const double* lr_dev) {
    return reduce_step(a, lr_dev);
  }

  static __device__ __forceinline__ float rule(const Args& a, const Step& s, float g, float w, float& b, bool decay) {
    if (a.maximize) g = -g;
    if (decay) g = fmaf(a.weight_decay, w, g);                     // grad.add(param, alpha=weight_decay)
    if (a.buf != nullptr) {
      // first step: buf = grad.clone(); then buf.mul_(momentum).add_(grad, alpha=1 - dampening)
      b = s.first ? g : fmaf(a.one_minus_dampening, g, __fmul_rn(b, a.momentum));
      g = a.nesterov ? fmaf(a.momentum, b, g) : b;                 // grad.add(buf, alpha=momentum) : buf
    }
    return fmaf(s.neg_lr, g, w);                                   // param.add_(grad, alpha=-lr)
  }

  template <class P>
  static __device__ __forceinline__ void update8(const P& p, const Step& s, long long e, const float* g,
                                                 float inv_world, float coef, bool decay, float* w) {
    const Args& a = p.rule;
    const float4 w0 = *reinterpret_cast<const float4*>(p.master + e);
    const float4 w1 = *reinterpret_cast<const float4*>(p.master + e + 4);
    w[0] = w0.x; w[1] = w0.y; w[2] = w0.z; w[3] = w0.w; w[4] = w1.x; w[5] = w1.y; w[6] = w1.z; w[7] = w1.w;
    float b[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (a.buf != nullptr && !s.first) {
      const float4 b0 = *reinterpret_cast<const float4*>(a.buf + e), b1 = *reinterpret_cast<const float4*>(a.buf + e + 4);
      b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) w[k] = rule(a, s, g[k] * inv_world * coef, w[k], b[k], decay);
    *reinterpret_cast<float4*>(p.master + e) = make_float4(w[0], w[1], w[2], w[3]);
    *reinterpret_cast<float4*>(p.master + e + 4) = make_float4(w[4], w[5], w[6], w[7]);
    if (a.buf != nullptr) {
      *reinterpret_cast<float4*>(a.buf + e) = make_float4(b[0], b[1], b[2], b[3]);
      *reinterpret_cast<float4*>(a.buf + e + 4) = make_float4(b[4], b[5], b[6], b[7]);
    }
  }

  template <class P>
  static __device__ __forceinline__ float4 update4(const P& p, const Step& s, long long e, uint2 q, float coef) {
    const Args& a = p.rule;
    float4 w = *reinterpret_cast<const float4*>(p.master + e);
    const bool decay = p.has_wd && p.decay[e >> 3];
    float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
    if (a.buf != nullptr && !s.first) b = *reinterpret_cast<const float4*>(a.buf + e);
    w.x = rule(a, s, bf16_lo(q.x) * coef, w.x, b.x, decay);
    w.y = rule(a, s, bf16_hi(q.x) * coef, w.y, b.y, decay);
    w.z = rule(a, s, bf16_lo(q.y) * coef, w.z, b.z, decay);
    w.w = rule(a, s, bf16_hi(q.y) * coef, w.w, b.w, decay);
    if (a.buf != nullptr) *reinterpret_cast<float4*>(a.buf + e) = b;
    *reinterpret_cast<float4*>(p.master + e) = w;
    return w;
  }
};

// torch.optim.Adam / AdamW with fused=True (torch 2.11 ATen/native/cuda/fused_adam_utils.cuh, `adam_math`), per
// element in fp32: the hyperparameters are the doubles cast to float, t is the float step count, and the two bias
// corrections are formed in float (torch_adam_bias_correction).  AMSGRAD is a template flag, so the update without it
// carries no max_exp_avg_sq traffic or registers; both slim instantiations fit in 32 registers with no spills.
__device__ __forceinline__ void torch_adam_bias_correction(float lr, float beta1, float beta2, long long step,
                                                           float* step_size, float* bc2_sqrt) {
  const float t = (float)(step + 1);
  *step_size = lr / (1.0f - powf(beta1, t));          // lr / bias_correction1
  *bc2_sqrt = sqrtf(1.0f - powf(beta2, t));
}

template <bool AMSGRAD>
struct TorchAdamRule {
  struct Args {
    float* m; float* v;
    float* vmax;                     // max_exp_avg_sq (AMSGRAD only)
    float lr, beta1, beta2, weight_decay, eps;   // static_cast<float> of the python doubles, as torch's opmath values
    int maximize, decoupled;         // decoupled: AdamW's decay of the weight; else Adam's L2 term in the gradient
    const long long* step_counter;   // reduce form: t = *step_counter + 1
    const float* prepared;           // slim form: {lr / bias_correction1, sqrt(bias_correction2)} from the prepare kernel
  };
  struct Step { float step_size, bc2_sqrt, lr_wd; };

  static __device__ __forceinline__ float lr_of(const Args& a, const double* lr_dev) {
    return lr_dev != nullptr ? (float)*lr_dev : a.lr;   // torch: static_cast<opmath_t>(lr)
  }
  static __device__ __forceinline__ Step reduce_step(const Args& a, const double* lr_dev) {
    Step s;
    const float lr = lr_of(a, lr_dev);
    torch_adam_bias_correction(lr, a.beta1, a.beta2, *a.step_counter, &s.step_size, &s.bc2_sqrt);
    s.lr_wd = lr * a.weight_decay;
    return s;
  }
  static __device__ __forceinline__ Step slim_step(const Args& a, const double* lr_dev) {
    return {a.prepared[0], a.prepared[1], lr_of(a, lr_dev) * a.weight_decay};
  }

  // adam_math on one element in three parts, so the slim form can store the moments before it holds the weights.
  // Each `a * b + c` is one fma and every other operation is rounded on its own, as in torch's build -- except Adam's
  // L2 term `grad += param * weight_decay`, which torch's build (sm_90 SASS of FusedAdamMathFunctor) forms as one fma
  // in the amsgrad kernel and whenever it unscales a GradScaler gradient, and otherwise as a product and a sum when
  // maximizing and in the first of the four elements a thread holds (lane 0), one fma in the other three.  A thread's
  // lanes are the elements 4i..4i+3 of a tensor whose size is a multiple of 4; a tensor of any other size goes through
  // torch's unaligned loop, where element j is in lane (j % 2048) / 512: its decay flags carry that (B2_ADAM_DECAY_*).
  static __device__ __forceinline__ bool l2_fma(const Args& a, bool scaled, bool lane0) {
    return AMSGRAD || scaled || !(a.maximize || lane0);
  }
  static __device__ __forceinline__ bool lane0(uint8_t flags, int k) {
    return (flags & B2_ADAM_DECAY_UNALIGNED) ? (flags & B2_ADAM_DECAY_LANE0) != 0 : (k & 3) == 0;
  }
  // grad: g the gradient of the shared path, w the master before the update
  static __device__ __forceinline__ float grad(const Args& a, float g, float w, bool decay, bool fma_l2) {
    if (a.maximize) g = -g;
    if (decay && !a.decoupled)                                     // grad += param * weight_decay
      g = fma_l2 ? fmaf(w, a.weight_decay, g) : __fadd_rn(g, __fmul_rn(w, a.weight_decay));
    return g;
  }
  // moments: g from grad(); m, v and vm (AMSGRAD) are updated in place.  Returns the second moment the denominator uses.
  static __device__ __forceinline__ float moments(const Args& a, float g, float& m, float& v, float& vm) {
    m = fmaf(a.beta1, m, fmaf(-a.beta1, g, g));
    const float g2 = __fmul_rn(g, g);
    v = fmaf(a.beta2, v, fmaf(-a.beta2, g2, g2));
    if (!AMSGRAD) return v;
    vm = vm < v ? v : vm;                                          // std::max(max_exp_avg_sq, exp_avg_sq)
    return vm;
  }
  // step_size * exp_avg / denom
  static __device__ __forceinline__ float direction(const Args& a, const Step& s, float m, float d) {
    const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(d), s.bc2_sqrt), a.eps);
    return __fdiv_rn(__fmul_rn(s.step_size, m), denom);
  }
  // the new master from the old one
  static __device__ __forceinline__ float weight(const Args& a, const Step& s, float w, float u, bool decay) {
    if (decay && a.decoupled) w = fmaf(-s.lr_wd, w, w);            // param -= lr * weight_decay * param
    return __fsub_rn(w, u);                                        // param -= step_size * exp_avg / denom
  }

  template <class P>
  static __device__ __forceinline__ void update8(const P& p, const Step& s, long long e, const float* g,
                                                 float inv_world, float coef, bool decay, float* w) {
    const Args& a = p.rule;
    float4 w0 = *reinterpret_cast<const float4*>(p.master + e), w1 = *reinterpret_cast<const float4*>(p.master + e + 4);
    float4 m0 = *reinterpret_cast<const float4*>(a.m + e), m1 = *reinterpret_cast<const float4*>(a.m + e + 4);
    float4 v0 = *reinterpret_cast<const float4*>(a.v + e), v1 = *reinterpret_cast<const float4*>(a.v + e + 4);
    w[0] = w0.x; w[1] = w0.y; w[2] = w0.z; w[3] = w0.w; w[4] = w1.x; w[5] = w1.y; w[6] = w1.z; w[7] = w1.w;
    float mm[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
    float vv[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
    float xx[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (AMSGRAD) {
      const float4 x0 = *reinterpret_cast<const float4*>(a.vmax + e), x1 = *reinterpret_cast<const float4*>(a.vmax + e + 4);
      xx[0] = x0.x; xx[1] = x0.y; xx[2] = x0.z; xx[3] = x0.w; xx[4] = x1.x; xx[5] = x1.y; xx[6] = x1.z; xx[7] = x1.w;
    }
    const uint8_t flags = decay ? p.decay[e >> 3] : 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const bool fma_l2 = l2_fma(a, p.grad_scale != nullptr, lane0(flags, k));
      const float d = moments(a, grad(a, g[k] * inv_world * coef, w[k], decay, fma_l2), mm[k], vv[k], xx[k]);
      w[k] = weight(a, s, w[k], direction(a, s, mm[k], d), decay);
    }
    *reinterpret_cast<float4*>(p.master + e) = make_float4(w[0], w[1], w[2], w[3]);
    *reinterpret_cast<float4*>(p.master + e + 4) = make_float4(w[4], w[5], w[6], w[7]);
    *reinterpret_cast<float4*>(a.m + e) = make_float4(mm[0], mm[1], mm[2], mm[3]);
    *reinterpret_cast<float4*>(a.m + e + 4) = make_float4(mm[4], mm[5], mm[6], mm[7]);
    *reinterpret_cast<float4*>(a.v + e) = make_float4(vv[0], vv[1], vv[2], vv[3]);
    *reinterpret_cast<float4*>(a.v + e + 4) = make_float4(vv[4], vv[5], vv[6], vv[7]);
    if (AMSGRAD) {
      *reinterpret_cast<float4*>(a.vmax + e) = make_float4(xx[0], xx[1], xx[2], xx[3]);
      *reinterpret_cast<float4*>(a.vmax + e + 4) = make_float4(xx[4], xx[5], xx[6], xx[7]);
    }
  }

  template <class P>
  static __device__ __forceinline__ float4 update4(const P& p, const Step& s, long long e, uint2 q, float coef) {
    const Args& a = p.rule;
    const uint8_t flags = p.has_wd ? p.decay[e >> 3] : 0;
    const bool decay = flags != 0;
    float4 mm, vv, d;
    if constexpr (AMSGRAD) {
      // the L2 term is always one fma here: the moments straight after the loads
      mm = *reinterpret_cast<const float4*>(a.m + e);
      vv = *reinterpret_cast<const float4*>(a.v + e);
      const float4 w = *reinterpret_cast<const float4*>(p.master + e);   // the coupled decay reads it
      float4 xx = *reinterpret_cast<const float4*>(a.vmax + e);
      d.x = moments(a, grad(a, bf16_lo(q.x) * coef, w.x, decay, true), mm.x, vv.x, xx.x);
      d.y = moments(a, grad(a, bf16_hi(q.x) * coef, w.y, decay, true), mm.y, vv.y, xx.y);
      d.z = moments(a, grad(a, bf16_lo(q.y) * coef, w.z, decay, true), mm.z, vv.z, xx.z);
      d.w = moments(a, grad(a, bf16_hi(q.y) * coef, w.w, decay, true), mm.w, vv.w, xx.w);
      *reinterpret_cast<float4*>(a.vmax + e) = xx;
    } else {
      // the gradients first, while the master weights are live, then the moments: fewer values live at once.  e is a
      // multiple of 4, so .x is the only element that can be in lane 0 of an aligned tensor (and this form has no
      // GradScaler state)
      float4 gg;
      {
        const float4 w = *reinterpret_cast<const float4*>(p.master + e);
        gg.x = grad(a, bf16_lo(q.x) * coef, w.x, decay, l2_fma(a, false, lane0(flags, 0)));
        gg.y = grad(a, bf16_hi(q.x) * coef, w.y, decay, l2_fma(a, false, lane0(flags, 1)));
        gg.z = grad(a, bf16_lo(q.y) * coef, w.z, decay, l2_fma(a, false, lane0(flags, 2)));
        gg.w = grad(a, bf16_hi(q.y) * coef, w.w, decay, l2_fma(a, false, lane0(flags, 3)));
      }
      mm = *reinterpret_cast<const float4*>(a.m + e);
      vv = *reinterpret_cast<const float4*>(a.v + e);
      float unused = 0.f;
      d.x = moments(a, gg.x, mm.x, vv.x, unused);
      d.y = moments(a, gg.y, mm.y, vv.y, unused);
      d.z = moments(a, gg.z, mm.z, vv.z, unused);
      d.w = moments(a, gg.w, mm.w, vv.w, unused);
    }
    *reinterpret_cast<float4*>(a.m + e) = mm;
    *reinterpret_cast<float4*>(a.v + e) = vv;
    // the directions first, then the master weights again (an L1 hit): fewer values live across the divisions
    float4 u;
    u.x = direction(a, s, mm.x, d.x);
    u.y = direction(a, s, mm.y, d.y);
    u.z = direction(a, s, mm.z, d.z);
    u.w = direction(a, s, mm.w, d.w);
    float4 w = *reinterpret_cast<const float4*>(p.master + e);
    w.x = weight(a, s, w.x, u.x, decay);
    w.y = weight(a, s, w.y, u.y, decay);
    w.z = weight(a, s, w.z, u.z, decay);
    w.w = weight(a, s, w.w, u.w, decay);
    *reinterpret_cast<float4*>(p.master + e) = w;
    return w;
  }
};

// ---- reduce form: any world ----------------------------------------------------------------------------------------
template <class Rule>
struct ReduceParams {
  const __nv_bfloat16* grads[MAX_WORLD];
  __nv_bfloat16* shadow[MAX_WORLD];
  int world;
  float* master;
  const uint8_t* decay;
  long long begin, end;  // element range, multiples of 8
  int has_wd;
  const float* grad_scale;   // optional device scalar (GradScaler): gradients are divided by it
  const float* found_inf;    // optional device scalar (GradScaler): non-zero skips the update
  const float* clip_coef;    // optional device scalar (gradient clipping): gradients are multiplied by it
  const float* grad_f32;     // optional fp32 mean gradient of [begin, end), indexed from begin: read instead of peers
  const double* lr_dev;      // optional device fp64 learning rate (a captured step's schedule): read instead of the lr
  typename Rule::Args rule;
};

template <class Rule>
__global__ void __launch_bounds__(256) reduce_update_kernel(const ReduceParams<Rule> p) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  if (p.found_inf != nullptr && *p.found_inf != 0.f) return;   // GradScaler saw inf/nan: this step is skipped
  // x * 1.0f is exact: without a coefficient the update is the unclipped one, bit for bit
  const float coef = p.clip_coef != nullptr ? *p.clip_coef : 1.0f;
  const typename Rule::Step s = Rule::reduce_step(p.rule, p.lr_dev);
  // mean over ranks (unless grad_f32 already holds it); with a GradScaler also the unscale (a power of two: exact)
  const float inv_world = (p.grad_scale != nullptr ? 1.0f / *p.grad_scale : 1.0f) /
                          (p.grad_f32 != nullptr ? 1.0f : (float)p.world);
  const long long nvec = (p.end - p.begin) >> 3;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * blockDim.x) {
    const long long e = p.begin + (i << 3);
    float g[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (p.grad_f32 != nullptr) {
      const float4 a0 = *reinterpret_cast<const float4*>(p.grad_f32 + (e - p.begin));
      const float4 a1 = *reinterpret_cast<const float4*>(p.grad_f32 + (e - p.begin) + 4);
      g[0] = a0.x; g[1] = a0.y; g[2] = a0.z; g[3] = a0.w; g[4] = a1.x; g[5] = a1.y; g[6] = a1.z; g[7] = a1.w;
    } else {
#pragma unroll
      for (int r = 0; r < MAX_WORLD; ++r) {
        if (r < p.world) {
          // peer-mapped pointer: plain 16-byte global load; the address aperture routes it over NVLink
          const uint4 q = *reinterpret_cast<const uint4*>(p.grads[r] + e);
          g[0] += bf16_lo(q.x); g[1] += bf16_hi(q.x); g[2] += bf16_lo(q.y); g[3] += bf16_hi(q.y);
          g[4] += bf16_lo(q.z); g[5] += bf16_hi(q.z); g[6] += bf16_lo(q.w); g[7] += bf16_hi(q.w);
        }
      }
    }
    const bool decay = p.has_wd && p.decay[e >> 3];
    float w[8];
    Rule::update8(p, s, e, g, inv_world, coef, decay, w);
    uint4 o;
    o.x = pack_bf16(w[0], w[1]); o.y = pack_bf16(w[2], w[3]);
    o.z = pack_bf16(w[4], w[5]); o.w = pack_bf16(w[6], w[7]);
#pragma unroll
    for (int r = 0; r < MAX_WORLD; ++r)
      if (r < p.world && p.shadow[r] != nullptr) *reinterpret_cast<uint4*>(p.shadow[r] + e) = o;
  }
}

// ---- single-GPU background form ------------------------------------------------------------------------------------
// On one GPU the optimizer kernels run on their own stream under the backward pass, but a 256-thread x 64-register
// block cannot become resident on an SM whose registers are held by a GEMM CTA, so the update only runs in the gaps
// between GEMM kernels.  This variant is shaped to fit beside such a CTA: 128 threads x 32 registers, no shared
// memory, and the same shared-memory carve-out preference as the GEMM kernels (an SM is not re-partitioned while it
// has resident CTAs).  Blocks are short-lived (8 vectors of 4 elements per thread) so they never hold an SM back from
// a kernel that needs all of it (the attention kernels).  Same arithmetic, statement for statement, as
// reduce_update_kernel with world == 1; for AdamW the bias-corrected step size is computed once per step by
// adamw_prepare_kernel (double pow, as the host would) instead of in every block.  The co-resident blocks are bound by
// the latency of their own dependent load -> sqrt -> divide -> store chain, not by HBM queue depth.
template <class Rule>
struct SlimParams {
  const __nv_bfloat16* grads; __nv_bfloat16* shadow;
  float* master;
  const uint8_t* decay;
  long long begin, nvec4;
  int has_wd;
  const float* clip_coef;   // optional (gradient clipping): gradients are multiplied by it
  const double* lr_dev;     // optional device fp64 learning rate
  typename Rule::Args rule;
};
constexpr int kSlimThreads = 128, kSlimIters = 8;
template <class Rule>
__global__ void __launch_bounds__(sizeof(Rule) > 0 ? kSlimThreads : 0) __maxnreg__(sizeof(Rule) > 0 ? 32 : 24)
slim_update_kernel(const SlimParams<Rule> p) {
  pdl_wait();
  pdl_launch_dependents();
  const typename Rule::Step s = Rule::slim_step(p.rule, p.lr_dev);
  const float coef = p.clip_coef != nullptr ? *p.clip_coef : 1.0f;   // x * 1.0f is exact
  long long i = (long long)blockIdx.x * (kSlimThreads * kSlimIters) + threadIdx.x;
#pragma unroll 1
  for (int it = 0; it < kSlimIters; ++it, i += kSlimThreads) {
    if (i >= p.nvec4) break;
    const long long e = p.begin + (i << 2);
    const uint2 q = *reinterpret_cast<const uint2*>(p.grads + e);
    const float4 w = Rule::update4(p, s, e, q, coef);
    uint2 o;
    o.x = pack_bf16(w.x, w.y);
    o.y = pack_bf16(w.z, w.w);
    *reinterpret_cast<uint2*>(p.shadow + e) = o;
  }
}

// ---- gradient accumulation -----------------------------------------------------------------------------------------
// One pass over [begin, end) of the bf16 gradient space and its fp32 accumulator (B2_ACCUM_* in the header).  It is
// launched per bucket on the optimizer stream while the backward's GEMM CTAs hold the SMs, so it has the shape of
// slim_update_kernel: 128 threads x <= 32 registers, no shared memory, the GEMMs' carve-out, short-lived blocks.  Each
// thread handles kAccIters vectors of 8 elements (16 bytes of bf16, 2 x float4 of fp32).  inf / nan pass through.
constexpr int kAccThreads = 128, kAccIters = 8;
template <int MODE>
__global__ void __maxnreg__(32)
grad_accumulate_kernel(__nv_bfloat16* __restrict__ grads, float* __restrict__ accum, long long begin, long long nvec) {
  pdl_wait();
  pdl_launch_dependents();
  long long i = (long long)blockIdx.x * (kAccThreads * kAccIters) + threadIdx.x;
#pragma unroll 1
  for (int it = 0; it < kAccIters; ++it, i += kAccThreads) {
    if (i >= nvec) break;
    const long long e = begin + (i << 3);
    float4* a = reinterpret_cast<float4*>(accum + e);
    uint4* g = reinterpret_cast<uint4*>(grads + e);
    float f[8];
    if (MODE != B2_ACCUM_FLUSH) {
      const uint4 q = *g;
      f[0] = bf16_lo(q.x); f[1] = bf16_hi(q.x); f[2] = bf16_lo(q.y); f[3] = bf16_hi(q.y);
      f[4] = bf16_lo(q.z); f[5] = bf16_hi(q.z); f[6] = bf16_lo(q.w); f[7] = bf16_hi(q.w);
    }
    if (MODE != B2_ACCUM_STORE) {
      const float4 a0 = a[0], a1 = a[1];
      if (MODE == B2_ACCUM_FLUSH) {
        f[0] = a0.x; f[1] = a0.y; f[2] = a0.z; f[3] = a0.w; f[4] = a1.x; f[5] = a1.y; f[6] = a1.z; f[7] = a1.w;
      } else {
        f[0] = a0.x + f[0]; f[1] = a0.y + f[1]; f[2] = a0.z + f[2]; f[3] = a0.w + f[3];
        f[4] = a1.x + f[4]; f[5] = a1.y + f[5]; f[6] = a1.z + f[6]; f[7] = a1.w + f[7];
      }
    }
    if (MODE == B2_ACCUM_STORE || MODE == B2_ACCUM_ADD) {
      a[0] = make_float4(f[0], f[1], f[2], f[3]);
      a[1] = make_float4(f[4], f[5], f[6], f[7]);
    } else {
      uint4 o;
      o.x = pack_bf16(f[0], f[1]); o.y = pack_bf16(f[2], f[3]);
      o.z = pack_bf16(f[4], f[5]); o.w = pack_bf16(f[6], f[7]);
      *g = o;
    }
  }
}

template <int MODE>
static int32_t launch_grad_accumulate(void* grads, float* accum, long long begin, long long nvec, cudaStream_t stream) {
  static bool attr = false;
  if (!attr) {   // same shared-memory carve-out as the GEMM CTAs it is meant to run beside
    B2_CUDA(cudaFuncSetAttribute(grad_accumulate_kernel<MODE>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                 cudaSharedmemCarveoutMaxShared));
    attr = true;
  }
  const long long per_block = (long long)kAccThreads * kAccIters;
  B2_LAUNCH(grad_accumulate_kernel<MODE>, (unsigned)((nvec + per_block - 1) / per_block), kAccThreads, 0, stream,
            (__nv_bfloat16*)grads, accum, begin, nvec);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

// ---- gradient-norm clipping ----------------------------------------------------------------------------------------
// Reduce phase of a clipped step over [begin, end): world > 1 reads the slice from every peer, sums in fp32 in rank
// order, multiplies by 1/world and stores the mean into the fp32 stash (the update reads it back instead of the
// peers); world 1 only reads.  Every warp writes the sum of squares of the (mean) gradients it saw into its own fp64
// slot: no atomics, so the norm is bit-reproducible.  At world 1 it runs per bucket under the backward, so it has the
// shape of grad_accumulate_kernel: 128 threads x <= 32 registers, no shared memory, short-lived blocks.
struct SumsqParams {
  const __nv_bfloat16* grads[MAX_WORLD];
  int world;
  float inv_world;
  float* stash;        // world > 1: fp32 [end - begin], indexed from begin
  double* partials;    // B2_SUMSQ_SLOTS(end - begin) slots, 4 per block
  long long begin, nvec;
};
constexpr int kSqThreads = 128, kSqIters = 8;
static_assert(kSqThreads * kSqIters * 8 == 8192 && kSqThreads / 32 == 4, "B2_SUMSQ_SLOTS in the header");
__global__ void __maxnreg__(32) grad_reduce_sumsq_kernel(const SumsqParams p) {
  pdl_wait();
  pdl_launch_dependents();
  long long i = (long long)blockIdx.x * (kSqThreads * kSqIters) + threadIdx.x;
  double acc = 0.0;
#pragma unroll 1
  for (int it = 0; it < kSqIters; ++it, i += kSqThreads) {
    if (i >= p.nvec) break;
    const long long e = p.begin + (i << 3);
    float g[8];
    if (p.world == 1) {
      const uint4 q = *reinterpret_cast<const uint4*>(p.grads[0] + e);
      g[0] = bf16_lo(q.x); g[1] = bf16_hi(q.x); g[2] = bf16_lo(q.y); g[3] = bf16_hi(q.y);
      g[4] = bf16_lo(q.z); g[5] = bf16_hi(q.z); g[6] = bf16_lo(q.w); g[7] = bf16_hi(q.w);
    } else {
      // the sum of reduce_update_kernel, from +0 in rank order: the stash holds exactly the gradient it would use
#pragma unroll
      for (int k = 0; k < 8; ++k) g[k] = 0.f;
#pragma unroll
      for (int r = 0; r < MAX_WORLD; ++r) {
        if (r < p.world) {
          const uint4 q = *reinterpret_cast<const uint4*>(p.grads[r] + e);
          g[0] += bf16_lo(q.x); g[1] += bf16_hi(q.x); g[2] += bf16_lo(q.y); g[3] += bf16_hi(q.y);
          g[4] += bf16_lo(q.z); g[5] += bf16_hi(q.z); g[6] += bf16_lo(q.w); g[7] += bf16_hi(q.w);
        }
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) g[k] *= p.inv_world;
      float4* s = reinterpret_cast<float4*>(p.stash + (e - p.begin));
      s[0] = make_float4(g[0], g[1], g[2], g[3]);
      s[1] = make_float4(g[4], g[5], g[6], g[7]);
    }
    float sq = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) sq = fmaf(g[k], g[k], sq);
    acc += (double)sq;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) p.partials[blockIdx.x * (kSqThreads / 32) + (threadIdx.x >> 5)] = acc;
}

constexpr int kFinThreads = 1024;
// Norm finalize: sum the slots in a fixed order (fp64).  mode 0: world 1, the norm of these slots.  mode 1: write this
// rank's share of the sum of squares to *total_norm (then exchanged, see b2_grad_norm_finalize).  mode 2: start from the
// rank mean of the shares in *clip_coef (x world).  Then total_norm = sqrt(sum) [/ grad_scale] and torch's coefficient.
__global__ void grad_norm_finalize_kernel(const double* __restrict__ partials, long long nslots, int mode, int world,
                                          float max_norm, const float* grad_scale, const float* found_inf,
                                          float* total_norm, float* clip_coef, float* skip) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ double red[kFinThreads];
  double s = 0.0;
  if (mode != 2) {
    for (long long i = threadIdx.x; i < nslots; i += blockDim.x) s += partials[i];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = kFinThreads / 2; o > 0; o >>= 1) {
      if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
      __syncthreads();
    }
    s = red[0];
  }
  if (threadIdx.x != 0) return;
  if (mode == 1) {
    *total_norm = (float)s;
    return;
  }
  if (mode == 2) s = (double)*clip_coef * (double)world;   // identical on every rank: the mean is
  float norm = (float)sqrt(s);
  if (grad_scale != nullptr) norm = norm / *grad_scale;
  // torch.nn.utils.clip_grads_with_norm_: clamp(max_norm / (total_norm + 1e-6), max=1); a NaN norm stays NaN
  const float q = max_norm / (norm + 1e-6f);
  *total_norm = norm;
  *clip_coef = q > 1.0f ? 1.0f : q;
  if (skip != nullptr)
    *skip = ((found_inf != nullptr && *found_inf != 0.f) || (grad_scale != nullptr && !isfinite(norm))) ? 1.f : 0.f;
}

// HF AdamW bias correction for the NEXT update: step_size = lr * sqrt(1 - b2^t) / (1 - b1^t), t = *step + 1; lr is
// *lr_dev when that is set
__global__ void adamw_prepare_kernel(double lr_arg, const double* lr_dev, double beta1, double beta2, int correct_bias,
                                     const long long* step, float* step_size) {
  pdl_wait();
  pdl_launch_dependents();
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    const double lr = lr_dev != nullptr ? *lr_dev : lr_arg;
    double ss = lr;
    if (correct_bias) {
      const long long t = *step + 1;
      ss = lr * sqrt(1.0 - pow(beta2, (double)t)) / (1.0 - pow(beta1, (double)t));
    }
    *step_size = (float)ss;
  }
}

// torch Adam's bias corrections for the NEXT update (t = *step + 1), read by the slim form: prepared[0] = lr / bc1,
// prepared[1] = sqrt(bc2); lr is (float)*lr_dev when that is set
__global__ void torch_adam_prepare_kernel(float lr_arg, const double* lr_dev, float beta1, float beta2,
                                          const long long* step, float* prepared) {
  pdl_wait();
  pdl_launch_dependents();
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    const float lr = lr_dev != nullptr ? (float)*lr_dev : lr_arg;
    torch_adam_bias_correction(lr, beta1, beta2, *step, &prepared[0], &prepared[1]);
  }
}

__global__ void step_advance_kernel(long long* step, unsigned long long* rng, const float* found_inf) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    if (step && !(found_inf != nullptr && *found_inf != 0.f)) *step += 1;
    if (rng) rng[1] += 1;
  }
}
__global__ void rng_seed_kernel(unsigned long long* rng, unsigned long long seed, unsigned long long step) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    rng[0] = seed;
    rng[1] = step;
  }
}

__global__ void cast_f32_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long n) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i + 8 <= n) {
    const float4 a = *reinterpret_cast<const float4*>(src + i), b = *reinterpret_cast<const float4*>(src + i + 4);
    uint4 o;
    o.x = pack_bf16(a.x, a.y); o.y = pack_bf16(a.z, a.w); o.z = pack_bf16(b.x, b.y); o.w = pack_bf16(b.z, b.w);
    stg16(dst + i, o);
  } else {
    for (long long k = i; k < n; ++k) dst[k] = __float2bfloat16_rn(src[k]);
  }
}
__global__ void cast_bf16_f32_kernel(const __nv_bfloat16* __restrict__ src, float* __restrict__ dst, long long n) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = __bfloat162float(src[i]);
}

// segments [n][3] = {src offset, dst offset, count}: dst(bf16) <- src(fp32); src <- 0.  grid = (ceil(max_count/256), n)
__global__ void accum_finish_kernel(float* __restrict__ src, __nv_bfloat16* __restrict__ dst,
                                    const long long* __restrict__ seg) {
  pdl_wait();
  pdl_launch_dependents();
  const long long so = seg[blockIdx.y * 3], d0 = seg[blockIdx.y * 3 + 1], cnt = seg[blockIdx.y * 3 + 2];
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cnt) {
    dst[d0 + i] = __float2bfloat16_rn(src[so + i]);
    src[so + i] = 0.f;
  }
}

}  // namespace b2

using namespace b2;

extern "C" int32_t b2_accum_finish(float* src, void* dst, const int64_t* segments, int64_t n_segments,
                                   int64_t max_count, void* stream_) {
  B2_REQUIRE(src && dst && segments && n_segments > 0 && max_count > 0, "accum_finish: bad args");
  dim3 grid((unsigned)((max_count + 255) / 256), (unsigned)n_segments);
  B2_LAUNCH(accum_finish_kernel, grid, 256, 0, stream_, src, (__nv_bfloat16*)dst, (const long long*)segments);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

// The launch every optimizer's reduce entry point shares: checks, the gradient-path fields of the params (HP is
// b2_adamw_hparams_t, b2_sgd_hparams_t or b2_adam_hparams_t, whose optional device fields have the same names), the grid.
template <class Rule, class HP>
static int32_t launch_reduce(const char* what, const void* const* peer_grads, void* const* peer_shadow, int32_t world,
                             int32_t rank, float* master, const uint8_t* decay_flags, int64_t begin, int64_t end,
                             const HP* hp, int has_wd, const typename Rule::Args& rule, void* stream_) {
  B2_REQUIRE(world >= 1 && world <= MAX_WORLD && rank >= 0 && rank < world, "%s: world=%d rank=%d", what, world, rank);
  B2_REQUIRE(begin >= 0 && end >= begin && begin % 8 == 0 && end % 8 == 0,
             "%s: slice [%lld,%lld) must be 8-element aligned", what, (long long)begin, (long long)end);
  if (end == begin) return 0;
  ReduceParams<Rule> p;
  for (int r = 0; r < MAX_WORLD; ++r) {
    p.grads[r] = r < world ? (const __nv_bfloat16*)peer_grads[r] : nullptr;
    p.shadow[r] = r < world ? (__nv_bfloat16*)peer_shadow[r] : nullptr;
    // a NULL shadow entry = that peer's copy is delivered some other way (copy-engine all-gather)
    if (r < world) B2_REQUIRE(p.grads[r] && (p.shadow[r] || r != rank), "%s: null peer pointer for rank %d", what, r);
  }
  p.world = world;
  p.master = master; p.decay = decay_flags;
  p.begin = begin; p.end = end;
  p.has_wd = has_wd;
  p.grad_scale = hp->grad_scale;
  p.found_inf = hp->found_inf;
  p.clip_coef = hp->clip_coef;
  p.grad_f32 = hp->grad_f32;
  p.lr_dev = hp->lr_dev;
  p.rule = rule;
  B2_REQUIRE((uintptr_t)p.grad_f32 % 16 == 0, "%s: grad_f32 must be 16-byte aligned", what);
  const long long nvec = (end - begin) >> 3;
  long long blocks = (nvec + 255) / 256;
  const long long cap = 132 * 8;   // 8 blocks per SM of an H100
  if (blocks > cap) blocks = cap;
  B2_LAUNCH(reduce_update_kernel<Rule>, (unsigned)blocks, 256, 0, (cudaStream_t)stream_, p);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

template <class Rule, class HP>
static int32_t launch_slim(const char* what, const void* grads, void* shadow, float* master,
                           const uint8_t* decay_flags, int64_t begin, int64_t end, const HP* hp, int has_wd,
                           const typename Rule::Args& rule, void* stream_) {
  B2_REQUIRE(begin >= 0 && end >= begin && begin % 8 == 0 && end % 8 == 0,
             "%s: slice [%lld,%lld) must be 8-element aligned", what, (long long)begin, (long long)end);
  B2_REQUIRE(hp->grad_scale == nullptr && hp->found_inf == nullptr && hp->grad_f32 == nullptr,
             "%s: GradScaler state and fp32 sources are handled by the bucket_reduce form", what);
  if (end == begin) return 0;
  static bool attr = false;
  if (!attr) {   // same shared-memory carve-out as the GEMM CTAs it is meant to run beside
    B2_CUDA(cudaFuncSetAttribute(slim_update_kernel<Rule>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                 cudaSharedmemCarveoutMaxShared));
    attr = true;
  }
  SlimParams<Rule> p;
  p.grads = (const __nv_bfloat16*)grads; p.shadow = (__nv_bfloat16*)shadow;
  p.master = master; p.decay = decay_flags;
  p.begin = begin; p.nvec4 = (end - begin) >> 2;
  p.has_wd = has_wd;
  p.clip_coef = hp->clip_coef;
  p.lr_dev = hp->lr_dev;
  p.rule = rule;
  const long long per_block = (long long)kSlimThreads * kSlimIters;
  const long long blocks = (p.nvec4 + per_block - 1) / per_block;
  B2_LAUNCH(slim_update_kernel<Rule>, (unsigned)blocks, kSlimThreads, 0, (cudaStream_t)stream_, p);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

static AdamWRule::Args adamw_args(const b2_adamw_hparams_t* hp, float* exp_avg, float* exp_avg_sq) {
  AdamWRule::Args a;
  a.m = exp_avg; a.v = exp_avg_sq;
  a.lr_d = hp->lr; a.beta1_d = hp->beta1; a.beta2_d = hp->beta2; a.weight_decay_d = hp->weight_decay;
  a.lr = (float)hp->lr; a.beta1 = (float)hp->beta1; a.beta2 = (float)hp->beta2;
  a.one_minus_beta1 = (float)(1.0 - hp->beta1); a.one_minus_beta2 = (float)(1.0 - hp->beta2);
  a.eps = (float)hp->eps; a.lr_wd = (float)(hp->lr * hp->weight_decay);
  a.correct_bias = hp->correct_bias;
  a.step_counter = nullptr;
  a.step_size = nullptr;
  return a;
}

extern "C" int32_t b2_bucket_reduce_adamw(const void* const* peer_grads, void* const* peer_shadow, int32_t world,
                                          int32_t rank, float* master, float* exp_avg, float* exp_avg_sq,
                                          const uint8_t* decay_flags, int64_t begin, int64_t end,
                                          const b2_adamw_hparams_t* hp, const int64_t* step_counter, void* stream_) {
  B2_REQUIRE(peer_grads && peer_shadow && master && exp_avg && exp_avg_sq && decay_flags && hp && step_counter,
             "bucket_reduce_adamw: null pointer");
  AdamWRule::Args a = adamw_args(hp, exp_avg, exp_avg_sq);
  a.step_counter = (const long long*)step_counter;
  return launch_reduce<AdamWRule>("bucket_reduce_adamw", peer_grads, peer_shadow, world, rank, master, decay_flags,
                                  begin, end, hp, hp->weight_decay > 0.0 ? 1 : 0, a, stream_);
}

extern "C" int32_t b2_adamw_prepare(const b2_adamw_hparams_t* hp, const int64_t* step_counter, float* step_size,
                                    void* stream_) {
  B2_REQUIRE(hp && step_counter && step_size, "adamw_prepare: null pointer");
  B2_LAUNCH(adamw_prepare_kernel, 1, 32, 0, (cudaStream_t)stream_, hp->lr, hp->lr_dev, hp->beta1, hp->beta2,
            hp->correct_bias, (const long long*)step_counter, step_size);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_adamw_background(const void* grads, void* shadow, float* master, float* exp_avg,
                                       float* exp_avg_sq, const uint8_t* decay_flags, int64_t begin, int64_t end,
                                       const b2_adamw_hparams_t* hp, const float* step_size, void* stream_) {
  B2_REQUIRE(grads && shadow && master && exp_avg && exp_avg_sq && decay_flags && hp && step_size,
             "adamw_background: null pointer");
  AdamWRule::Args a = adamw_args(hp, exp_avg, exp_avg_sq);
  a.step_size = step_size;
  return launch_slim<AdamWRule>("adamw_background", grads, shadow, master, decay_flags, begin, end, hp,
                                hp->weight_decay > 0.0 ? 1 : 0, a, stream_);
}

// the buffer is there exactly when the update uses one; the step counter tells its first step
static int32_t sgd_args(const char* what, const b2_sgd_hparams_t* hp, float* momentum_buffer,
                        const int64_t* step_counter, SgdRule::Args* a) {
  B2_REQUIRE((hp->momentum != 0.0) == (momentum_buffer != nullptr),
             "%s: momentum_buffer must be given exactly when momentum != 0 (momentum=%g)", what, hp->momentum);
  B2_REQUIRE(momentum_buffer == nullptr || step_counter != nullptr, "%s: step_counter is required with momentum", what);
  B2_REQUIRE(!hp->nesterov || (hp->momentum > 0.0 && hp->dampening == 0.0),
             "%s: Nesterov momentum requires a momentum and zero dampening", what);
  a->buf = momentum_buffer;
  a->step_counter = (const long long*)step_counter;
  a->neg_lr = (float)(-hp->lr);
  a->momentum = (float)hp->momentum;
  a->one_minus_dampening = (float)(1.0 - hp->dampening);
  a->weight_decay = (float)hp->weight_decay;
  a->nesterov = hp->nesterov ? 1 : 0;
  a->maximize = hp->maximize ? 1 : 0;
  return 0;
}

extern "C" int32_t b2_bucket_reduce_sgd(const void* const* peer_grads, void* const* peer_shadow, int32_t world,
                                        int32_t rank, float* master, float* momentum_buffer,
                                        const uint8_t* decay_flags, int64_t begin, int64_t end,
                                        const b2_sgd_hparams_t* hp, const int64_t* step_counter, void* stream_) {
  B2_REQUIRE(peer_grads && peer_shadow && master && decay_flags && hp, "bucket_reduce_sgd: null pointer");
  SgdRule::Args a;
  const int32_t st = sgd_args("bucket_reduce_sgd", hp, momentum_buffer, step_counter, &a);
  if (st) return st;
  return launch_reduce<SgdRule>("bucket_reduce_sgd", peer_grads, peer_shadow, world, rank, master, decay_flags, begin,
                                end, hp, hp->weight_decay != 0.0 ? 1 : 0, a, stream_);
}

extern "C" int32_t b2_sgd_background(const void* grads, void* shadow, float* master, float* momentum_buffer,
                                     const uint8_t* decay_flags, int64_t begin, int64_t end,
                                     const b2_sgd_hparams_t* hp, const int64_t* step_counter, void* stream_) {
  B2_REQUIRE(grads && shadow && master && decay_flags && hp, "sgd_background: null pointer");
  SgdRule::Args a;
  const int32_t st = sgd_args("sgd_background", hp, momentum_buffer, step_counter, &a);
  if (st) return st;
  return launch_slim<SgdRule>("sgd_background", grads, shadow, master, decay_flags, begin, end, hp,
                              hp->weight_decay != 0.0 ? 1 : 0, a, stream_);
}

// the max_exp_avg_sq buffer is there exactly when the update is amsgrad's
template <bool AMSGRAD>
static int32_t torch_adam_args(const char* what, const b2_adam_hparams_t* hp, float* exp_avg, float* exp_avg_sq,
                               float* max_exp_avg_sq, typename TorchAdamRule<AMSGRAD>::Args* a) {
  B2_REQUIRE(exp_avg && exp_avg_sq, "%s: null moment pointer", what);
  B2_REQUIRE((hp->amsgrad != 0) == (max_exp_avg_sq != nullptr),
             "%s: max_exp_avg_sq must be given exactly when amsgrad is set (amsgrad=%d)", what, (int)hp->amsgrad);
  a->m = exp_avg; a->v = exp_avg_sq; a->vmax = max_exp_avg_sq;
  a->lr = (float)hp->lr; a->beta1 = (float)hp->beta1; a->beta2 = (float)hp->beta2;
  a->weight_decay = (float)hp->weight_decay; a->eps = (float)hp->eps;
  a->maximize = hp->maximize ? 1 : 0;
  a->decoupled = hp->decoupled ? 1 : 0;
  a->step_counter = nullptr;
  a->prepared = nullptr;
  return 0;
}

template <bool AMSGRAD>
static int32_t bucket_reduce_adam(const void* const* peer_grads, void* const* peer_shadow, int32_t world, int32_t rank,
                                  float* master, float* exp_avg, float* exp_avg_sq, float* max_exp_avg_sq,
                                  const uint8_t* decay_flags, int64_t begin, int64_t end, const b2_adam_hparams_t* hp,
                                  const int64_t* step_counter, void* stream_) {
  typename TorchAdamRule<AMSGRAD>::Args a;
  const int32_t st = torch_adam_args<AMSGRAD>("bucket_reduce_adam", hp, exp_avg, exp_avg_sq, max_exp_avg_sq, &a);
  if (st) return st;
  a.step_counter = (const long long*)step_counter;
  return launch_reduce<TorchAdamRule<AMSGRAD>>("bucket_reduce_adam", peer_grads, peer_shadow, world, rank, master,
                                               decay_flags, begin, end, hp, hp->weight_decay != 0.0 ? 1 : 0, a,
                                               stream_);
}

extern "C" int32_t b2_bucket_reduce_adam(const void* const* peer_grads, void* const* peer_shadow, int32_t world,
                                         int32_t rank, float* master, float* exp_avg, float* exp_avg_sq,
                                         float* max_exp_avg_sq, const uint8_t* decay_flags, int64_t begin, int64_t end,
                                         const b2_adam_hparams_t* hp, const int64_t* step_counter, void* stream_) {
  B2_REQUIRE(peer_grads && peer_shadow && master && decay_flags && hp && step_counter,
             "bucket_reduce_adam: null pointer");
  return hp->amsgrad ? bucket_reduce_adam<true>(peer_grads, peer_shadow, world, rank, master, exp_avg, exp_avg_sq,
                                                max_exp_avg_sq, decay_flags, begin, end, hp, step_counter, stream_)
                     : bucket_reduce_adam<false>(peer_grads, peer_shadow, world, rank, master, exp_avg, exp_avg_sq,
                                                 max_exp_avg_sq, decay_flags, begin, end, hp, step_counter, stream_);
}

extern "C" int32_t b2_adam_prepare(const b2_adam_hparams_t* hp, const int64_t* step_counter, float* prepared,
                                   void* stream_) {
  B2_REQUIRE(hp && step_counter && prepared, "adam_prepare: null pointer");
  B2_LAUNCH(torch_adam_prepare_kernel, 1, 32, 0, (cudaStream_t)stream_, (float)hp->lr, hp->lr_dev, (float)hp->beta1,
            (float)hp->beta2, (const long long*)step_counter, prepared);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_adam_background(const void* grads, void* shadow, float* master, float* exp_avg,
                                      float* exp_avg_sq, float* max_exp_avg_sq, const uint8_t* decay_flags,
                                      int64_t begin, int64_t end, const b2_adam_hparams_t* hp, const float* prepared,
                                      void* stream_) {
  B2_REQUIRE(grads && shadow && master && decay_flags && hp && prepared, "adam_background: null pointer");
  if (hp->amsgrad) {
    typename TorchAdamRule<true>::Args a;
    const int32_t st = torch_adam_args<true>("adam_background", hp, exp_avg, exp_avg_sq, max_exp_avg_sq, &a);
    if (st) return st;
    a.prepared = prepared;
    return launch_slim<TorchAdamRule<true>>("adam_background", grads, shadow, master, decay_flags, begin, end, hp,
                                            hp->weight_decay != 0.0 ? 1 : 0, a, stream_);
  }
  typename TorchAdamRule<false>::Args a;
  const int32_t st = torch_adam_args<false>("adam_background", hp, exp_avg, exp_avg_sq, max_exp_avg_sq, &a);
  if (st) return st;
  a.prepared = prepared;
  return launch_slim<TorchAdamRule<false>>("adam_background", grads, shadow, master, decay_flags, begin, end, hp,
                                           hp->weight_decay != 0.0 ? 1 : 0, a, stream_);
}

extern "C" int32_t b2_grad_accumulate(void* grads, float* accum, int64_t begin, int64_t end, int32_t mode,
                                      void* stream_) {
  B2_REQUIRE(grads && accum, "grad_accumulate: null pointer");
  B2_REQUIRE(((uintptr_t)grads % 16 == 0) && ((uintptr_t)accum % 16 == 0),
             "grad_accumulate: 16-byte alignment required");
  B2_REQUIRE(begin >= 0 && end >= begin && begin % 8 == 0 && end % 8 == 0,
             "grad_accumulate: slice [%lld,%lld) must be 8-element aligned", (long long)begin, (long long)end);
  B2_REQUIRE(mode >= B2_ACCUM_STORE && mode <= B2_ACCUM_FLUSH, "grad_accumulate: unknown mode %d", (int)mode);
  if (end == begin) return 0;
  const long long nvec = (end - begin) >> 3;
  cudaStream_t s = (cudaStream_t)stream_;
  switch (mode) {
    case B2_ACCUM_STORE: return launch_grad_accumulate<B2_ACCUM_STORE>(grads, accum, begin, nvec, s);
    case B2_ACCUM_ADD: return launch_grad_accumulate<B2_ACCUM_ADD>(grads, accum, begin, nvec, s);
    case B2_ACCUM_FOLD: return launch_grad_accumulate<B2_ACCUM_FOLD>(grads, accum, begin, nvec, s);
    default: return launch_grad_accumulate<B2_ACCUM_FLUSH>(grads, accum, begin, nvec, s);
  }
}

extern "C" int32_t b2_grad_reduce_sumsq(const void* const* peer_grads, int32_t world, float* stash, int64_t begin,
                                        int64_t end, double* partials, void* stream_) {
  B2_REQUIRE(peer_grads && partials, "grad_reduce_sumsq: null pointer");
  B2_REQUIRE(world >= 1 && world <= MAX_WORLD, "grad_reduce_sumsq: world=%d", world);
  B2_REQUIRE((world == 1) == (stash == nullptr), "grad_reduce_sumsq: the fp32 stash is required at world > 1 only");
  B2_REQUIRE(begin >= 0 && end >= begin && begin % 8 == 0 && end % 8 == 0,
             "grad_reduce_sumsq: slice [%lld,%lld) must be 8-element aligned", (long long)begin, (long long)end);
  B2_REQUIRE((uintptr_t)stash % 16 == 0, "grad_reduce_sumsq: 16-byte alignment required");
  if (end == begin) return 0;
  SumsqParams p;
  for (int r = 0; r < MAX_WORLD; ++r) {
    p.grads[r] = r < world ? (const __nv_bfloat16*)peer_grads[r] : nullptr;
    if (r < world) B2_REQUIRE(p.grads[r], "grad_reduce_sumsq: null peer pointer for rank %d", r);
  }
  p.world = world;
  p.inv_world = 1.0f / (float)world;
  p.stash = stash;
  p.partials = partials;
  p.begin = begin;
  p.nvec = (end - begin) >> 3;
  static bool attr = false;
  if (!attr) {   // same shared-memory carve-out as the GEMM CTAs it is meant to run beside
    B2_CUDA(cudaFuncSetAttribute(grad_reduce_sumsq_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                 cudaSharedmemCarveoutMaxShared));
    attr = true;
  }
  const long long per_block = (long long)kSqThreads * kSqIters;
  B2_LAUNCH(grad_reduce_sumsq_kernel, (unsigned)((p.nvec + per_block - 1) / per_block), kSqThreads, 0,
            (cudaStream_t)stream_, p);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_grad_norm_finalize(const double* partials, int64_t nslots, float* const* peer_scratch,
                                         void* const* peer_flags, int32_t world, int32_t rank, int32_t slot,
                                         uint32_t* epoch, float max_norm, const float* grad_scale,
                                         const float* found_inf, float* total_norm, float* clip_coef, float* skip,
                                         void* stream_) {
  B2_REQUIRE(partials && nslots >= 0 && total_norm && clip_coef, "grad_norm_finalize: bad args");
  B2_REQUIRE(world >= 1 && world <= MAX_WORLD && rank >= 0 && rank < world, "grad_norm_finalize: world=%d rank=%d",
             world, rank);
  cudaStream_t s = (cudaStream_t)stream_;
  if (world == 1) {
    B2_LAUNCH(grad_norm_finalize_kernel, 1, kFinThreads, 0, s, partials, (long long)nslots, 0, 1, max_norm, grad_scale,
              found_inf, total_norm, clip_coef, skip);
    B2_CUDA(cudaGetLastError());
    count_launches(1);
    return 0;
  }
  // the exchange's arguments are checked before the share kernel runs: a rejected call leaves *total_norm untouched
  B2_REQUIRE(peer_scratch && peer_flags && epoch, "grad_norm_finalize: null pointer");
  B2_REQUIRE(slot >= 0 && slot < B2_FLAG_SLOTS, "grad_norm_finalize: slot=%d", slot);
  for (int r = 0; r < world; ++r)
    B2_REQUIRE(peer_scratch[r] && peer_flags[r], "grad_norm_finalize: null peer pointer for rank %d", r);
  // this rank's share -> *total_norm; rank-order mean of the shares -> *clip_coef; then the norm from that mean
  B2_LAUNCH(grad_norm_finalize_kernel, 1, kFinThreads, 0, s, partials, (long long)nslots, 1, world, max_norm, grad_scale,
            found_inf, total_norm, clip_coef, skip);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  const int32_t st = b2_scalar_allreduce_mean(total_norm, clip_coef, peer_scratch, peer_flags, world, rank, slot,
                                              epoch, stream_);
  if (st) return st;
  B2_LAUNCH(grad_norm_finalize_kernel, 1, kFinThreads, 0, s, partials, (long long)nslots, 2, world, max_norm, grad_scale,
            found_inf, total_norm, clip_coef, skip);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_step_advance(int64_t* step_counter, void* rng_state, const float* found_inf, void* stream_) {
  B2_LAUNCH(step_advance_kernel, 1, 32, 0, (cudaStream_t)stream_, (long long*)step_counter,
            (unsigned long long*)rng_state, found_inf);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_rng_seed(void* rng_state, uint64_t seed, uint64_t step, void* stream_) {
  B2_REQUIRE(rng_state, "rng_seed: null pointer");
  B2_LAUNCH(rng_seed_kernel, 1, 32, 0, (cudaStream_t)stream_, (unsigned long long*)rng_state, seed, step);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_cast_f32_to_bf16(const float* src, void* dst, int64_t n, void* stream_) {
  B2_REQUIRE(src && dst && n >= 0, "cast_f32_to_bf16: bad args");
  B2_REQUIRE(((uintptr_t)src % 16 == 0) && ((uintptr_t)dst % 16 == 0), "cast_f32_to_bf16: 16-byte alignment required");
  if (n == 0) return 0;
  const long long nv = (n + 7) / 8;
  B2_LAUNCH(cast_f32_bf16_kernel, (unsigned)((nv + 255) / 256), 256, 0, (cudaStream_t)stream_, src, (__nv_bfloat16*)dst, n);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_cast_bf16_to_f32(const void* src, float* dst, int64_t n, void* stream_) {
  B2_REQUIRE(src && dst && n >= 0, "cast_bf16_to_f32: bad args");
  if (n == 0) return 0;
  B2_LAUNCH(cast_bf16_f32_kernel, (unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream_, (const __nv_bfloat16*)src, dst,
                                                                                       n);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_zero(void* dst, int64_t bytes, void* stream_) {
  B2_REQUIRE(dst && bytes >= 0, "zero: bad args");
  if (bytes == 0) return 0;
  B2_CUDA(cudaMemsetAsync(dst, 0, (size_t)bytes, (cudaStream_t)stream_));
  return 0;
}

extern "C" int32_t b2_copy_async(void* dst, const void* src, int64_t bytes, void* stream_) {
  B2_REQUIRE(dst && src && bytes >= 0, "copy_async: bad args");
  if (bytes == 0) return 0;
  // device-to-device: between a local buffer and an IPC-mapped peer buffer this is a copy-engine transfer over
  // NVLink that runs beside the SM kernels of other streams (a memcpy node when captured in a graph)
  B2_CUDA(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream_));
  return 0;
}
