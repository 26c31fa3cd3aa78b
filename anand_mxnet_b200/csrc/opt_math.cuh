// opt_math.cuh -- per-element optimizer arithmetic shared by the dense and row_sparse kernels.
//
// IEEE fp32, round-to-nearest, NO fused multiply-add: every operation is an explicit __f*_rn
// intrinsic (which the compiler never contracts), so results are bit-identical to the reference's
// CPU build and to oracle/kvoracle.c. Each branch cites the reference expression tree it follows.
#pragma once
#include "kernels.h"

namespace b200kv {

struct Hyper {
  float lr, wd, momentum, rescale, clip, beta1, beta2, eps;
};

// mshadow_op::clip (src/operator/mshadow_op.h:912-922)
__device__ __forceinline__ float clipf(float x, float b) { return x > b ? b : (x < -b ? -b : x); }

template <int OPT>
__device__ __forceinline__ float step(float w, float g, float& s1, float& s2, bool has_mom,
                                      const Hyper& h) {
  if (OPT == kOptAssign) {
    return g;
  } else if (OPT == kOptSGD) {
    // MultiSGDKernel / SGDMomKernel / MP_SGDMomKernel / SGDMomDnsRspDnsKernel
    // (optimizer_op-inl.h:232-254, 607-617, 706-724, 749-773)
    //   mom = momentum*mom - lr*wd*w - lr*rescale*g        | ... - lr*clip(rescale*g, c)
    //   w   = w + mom
    const float m0 = has_mom ? s1 : 0.f;
    const float a = __fsub_rn(__fmul_rn(h.momentum, m0), __fmul_rn(__fmul_rn(h.lr, h.wd), w));
    float m1;
    if (h.clip >= 0.f) {
      m1 = __fsub_rn(a, __fmul_rn(h.lr, clipf(__fmul_rn(h.rescale, g), h.clip)));
    } else {
      m1 = __fsub_rn(a, __fmul_rn(__fmul_rn(h.lr, h.rescale), g));
    }
    if (has_mom) s1 = m1;
    return __fadd_rn(w, m1);
  } else if (OPT == kOptSGDSingle) {
    // SGDKernel / MP_SGDKernel / SGDDnsRspKernel (optimizer_op-inl.h:388-397, 661-674, 453-475)
    //   w = (1-lr*wd)*w - (lr*rescale)*g                   | ... - lr*clip(rescale*g, c)
    const float a = __fmul_rn(__fsub_rn(1.f, __fmul_rn(h.lr, h.wd)), w);
    if (h.clip >= 0.f) {
      return __fsub_rn(a, __fmul_rn(h.lr, clipf(__fmul_rn(h.rescale, g), h.clip)));
    }
    return __fsub_rn(a, __fmul_rn(__fmul_rn(h.lr, h.rescale), g));
  } else if (OPT == kOptAdam) {
    // AdamUpdateKernel (optimizer_op-inl.h:1302-1312)
    float gr = __fadd_rn(__fmul_rn(g, h.rescale), __fmul_rn(w, h.wd));
    if (h.clip >= 0.f) gr = clipf(gr, h.clip);
    s1 = __fadd_rn(__fmul_rn(h.beta1, s1), __fmul_rn(__fsub_rn(1.f, h.beta1), gr));
    s2 = __fadd_rn(__fmul_rn(h.beta2, s2), __fmul_rn(__fmul_rn(__fsub_rn(1.f, h.beta2), gr), gr));
    return __fsub_rn(w, __fdiv_rn(__fmul_rn(h.lr, s1), __fadd_rn(__fsqrt_rn(s2), h.eps)));
  } else if (OPT == kOptTest) {
    // optimizer.py:2044-2046: weight[:] += grad * rescale_grad
    return __fadd_rn(w, __fmul_rn(g, h.rescale));
  }
  return w;
}

// AdamDnsRspDnsKernel<req,cpu> (optimizer_op-inl.h:1350-1380): the lazy CPU kernel squares the
// CLIPPED value first -- (1-beta2)*(c*c) -- unlike the dense kernel's ((1-beta2)*g)*g; without
// clipping both agree. The oracle is the CPU path, so the row_sparse kernel follows it.
__device__ __forceinline__ float step_adam_lazy(float w, float g, float& s1, float& s2,
                                                const Hyper& h) {
  const float gr = __fadd_rn(__fmul_rn(g, h.rescale), __fmul_rn(w, h.wd));
  if (h.clip >= 0.f) {
    const float c = clipf(gr, h.clip);
    s1 = __fadd_rn(__fmul_rn(h.beta1, s1), __fmul_rn(__fsub_rn(1.f, h.beta1), c));
    s2 = __fadd_rn(__fmul_rn(h.beta2, s2), __fmul_rn(__fsub_rn(1.f, h.beta2), __fmul_rn(c, c)));
  } else {
    s1 = __fadd_rn(__fmul_rn(h.beta1, s1), __fmul_rn(__fsub_rn(1.f, h.beta1), gr));
    s2 = __fadd_rn(__fmul_rn(h.beta2, s2), __fmul_rn(__fmul_rn(__fsub_rn(1.f, h.beta2), gr), gr));
  }
  return __fsub_rn(w, __fdiv_rn(__fmul_rn(h.lr, s1), __fadd_rn(__fsqrt_rn(s2), h.eps)));
}

// AdamStdDnsRspDnsKernel<req,cpu> (optimizer_op.cc:195-229): absent rows use g' = w*wd, and the
// variance squares first -- (1-beta2)*(g'*g') -- with or without clipping
__device__ __forceinline__ float step_adam_std(float w, float g, bool present, float& s1, float& s2,
                                               const Hyper& h) {
  float gr = present ? __fadd_rn(__fmul_rn(g, h.rescale), __fmul_rn(w, h.wd)) : __fmul_rn(w, h.wd);
  if (h.clip >= 0.f) gr = clipf(gr, h.clip);
  s1 = __fadd_rn(__fmul_rn(h.beta1, s1), __fmul_rn(__fsub_rn(1.f, h.beta1), gr));
  s2 = __fadd_rn(__fmul_rn(h.beta2, s2), __fmul_rn(__fsub_rn(1.f, h.beta2), __fmul_rn(gr, gr)));
  return __fsub_rn(w, __fdiv_rn(__fmul_rn(h.lr, s1), __fadd_rn(__fsqrt_rn(s2), h.eps)));
}

// ---- the single-tensor operators of the callback route: the dense elementwise kernel
// (update_kernels.cu) and the row-gather kernel of their row_sparse forms (rowsparse_kernels.cu)

// fp32 state arrays of each operator (input order after weight, grad) and whether it reads weight
__host__ __device__ constexpr int NumStates(int op) {
  return (op == kUpdSignSGD || op == kUpdSGD || op == kUpdSGDStd) ? 0
         : (op == kUpdNAG || op == kUpdSignum || op == kUpdRMSProp || op == kUpdAdaGrad || op == kUpdSGDMom) ? 1
         : (op == kUpdMPNAG || op == kUpdFtrl || op == kUpdAdamLazy || op == kUpdAdamStd) ? 2 : 3;
}
__host__ __device__ constexpr bool ReadsWeight(int op) { return op != kUpdMPNAG; }

// (x > 0) - (x < 0): an int, 0 for NaN
__device__ __forceinline__ float SignInt(float x) { return static_cast<float>((x > 0.f) - (x < 0.f)); }

// One element. w: weight (unused by mp_nag), g: gradient, s: the states, updated in place.
// present: the element's row is stored in a row_sparse gradient (g is +0.0f when it is not); only
// the standard sgd_update / adam_update forms tell the two apart. Returns the value stored to out.
template <int OP>
__device__ __forceinline__ float Step(const UpdateLaunch& a, float w, float g, float (&s)[3],
                                      bool present = true) {
  if (OP == kUpdSGD || OP == kUpdSGDStd || OP == kUpdSGDMom || OP == kUpdAdamLazy || OP == kUpdAdamStd) {
    const Hyper h{a.lr, a.wd, a.momentum, a.rescale, a.clip, a.beta1, a.beta2, a.eps};
    if (OP == kUpdSGD) return step<kOptSGDSingle>(w, g, s[0], s[1], false, h);
    if (OP == kUpdSGDMom) return step<kOptSGD>(w, g, s[0], s[1], true, h);  // g = +0.0f when absent
    if (OP == kUpdAdamLazy) return step_adam_lazy(w, g, s[0], s[1], h);
    if (OP == kUpdAdamStd) return step_adam_std(w, g, present, s[0], s[1], h);
    // standard sgd_update: the whole weight is scaled by (1 - lr*wd); present rows then take the
    // SGDDnsRspKernel step with wd = 0, i.e. (1.f - lr*0.f)*w' - ... = w' - ...
    const float scaled = __fmul_rn(w, __fsub_rn(1.f, __fmul_rn(h.lr, h.wd)));
    if (!present) return scaled;
    if (h.clip >= 0.f) return __fsub_rn(scaled, __fmul_rn(h.lr, clipf(__fmul_rn(h.rescale, g), h.clip)));
    return __fsub_rn(scaled, __fmul_rn(__fmul_rn(h.lr, h.rescale), g));
  }
  if (OP == kUpdNAG || OP == kUpdMPNAG) {
    // NAGMomKernel / MP_NAGMomKernel (optimizer_op-inl.h:1061-1138): mom = momentum*mom first;
    // out = (w - mom) + (momentum+1)*(mom - lr*(clip(rescale*g) + wd*w)); then
    // mom = mom - lr*(clip(rescale*g) + wd*w') where w' is the weight as it reads after out was
    // stored: the new value for mp_nag (a local) and for nag when out is the weight itself
    const float w0 = OP == kUpdMPNAG ? s[1] : w;
    float cg = __fmul_rn(a.rescale, g);
    if (a.clip >= 0.f) cg = clipf(cg, a.clip);
    const float mom = __fmul_rn(a.momentum, s[0]);
    const float out = __fadd_rn(__fsub_rn(w0, mom),
                                __fmul_rn(__fadd_rn(a.momentum, 1.f),
                                          __fsub_rn(mom, __fmul_rn(a.lr, __fadd_rn(cg, __fmul_rn(a.wd, w0))))));
    const float w1 = (OP == kUpdMPNAG || a.out_is_w) ? out : w0;
    s[0] = __fsub_rn(mom, __fmul_rn(a.lr, __fadd_rn(cg, __fmul_rn(a.wd, w1))));
    if (OP == kUpdMPNAG) s[1] = out;
    return out;
  }
  if (OP == kUpdSignSGD) {
    // SignSGDKernel (2344-2356): clip_gradient and rescale_grad have no effect
    return __fsub_rn(__fmul_rn(__fsub_rn(1.f, __fmul_rn(a.lr, a.wd)), w), __fmul_rn(a.lr, SignInt(g)));
  }
  if (OP == kUpdSignum) {
    // SignumKernel (2412-2431): the clipped branch multiplies (1-momentum) by clip(rescale*g), the
    // other one ((1-momentum)*rescale)*g
    const float om = __fsub_rn(1.f, a.momentum);
    const float t = a.clip >= 0.f ? __fmul_rn(om, clipf(__fmul_rn(a.rescale, g), a.clip))
                                  : __fmul_rn(__fmul_rn(om, a.rescale), g);
    s[0] = __fsub_rn(__fsub_rn(__fmul_rn(a.momentum, s[0]), __fmul_rn(__fmul_rn(om, a.wd), w)), t);
    return __fadd_rn(__fmul_rn(__fsub_rn(1.f, __fmul_rn(a.lr, a.wd_lh)), w), __fmul_rn(a.lr, SignInt(s[0])));
  }
  if (OP == kUpdRMSProp || OP == kUpdRMSPropAlex) {
    // RMSPropUpdateKernel (2052-2077), RMSPropAlexUpdateKernel (1953-1986): wd*w joins the
    // gradient before the clip
    float gr = __fadd_rn(__fmul_rn(a.rescale, g), __fmul_rn(a.wd, w));
    if (a.clip >= 0.f) gr = clipf(gr, a.clip);
    const float om = __fsub_rn(1.f, a.gamma1);
    float r;
    if (OP == kUpdRMSProp) {
      s[0] = __fadd_rn(__fmul_rn(om, __fmul_rn(gr, gr)), __fmul_rn(a.gamma1, s[0]));
      r = __fsub_rn(w, __fmul_rn(a.lr, __fdiv_rn(gr, __fsqrt_rn(__fadd_rn(s[0], a.eps)))));
    } else {
      s[0] = __fadd_rn(__fmul_rn(__fmul_rn(om, gr), gr), __fmul_rn(a.gamma1, s[0]));
      s[1] = __fadd_rn(__fmul_rn(om, gr), __fmul_rn(a.gamma1, s[1]));
      s[2] = __fsub_rn(__fmul_rn(a.gamma2, s[2]),
                       __fdiv_rn(__fmul_rn(a.lr, gr),
                                 __fsqrt_rn(__fadd_rn(__fsub_rn(s[0], __fmul_rn(s[1], s[1])), a.eps))));
      r = __fadd_rn(w, s[2]);
    }
    return a.clip_weights >= 0.f ? clipf(r, a.clip_weights) : r;
  }
  if (OP == kUpdFTML) {
    // FTMLKernel (1205-1222), states d, v, z; p1 = powf(beta1, t), p2 = powf(beta2, t)
    float gi = __fadd_rn(__fmul_rn(a.rescale, g), __fmul_rn(a.wd, w));
    if (a.clip >= 0.f) gi = clipf(gi, a.clip);
    s[1] = __fadd_rn(__fmul_rn(a.beta2, s[1]), __fmul_rn(__fsub_rn(1.f, a.beta2), __fmul_rn(gi, gi)));
    const float dt = __fmul_rn(__fdiv_rn(__fsub_rn(1.f, a.p1), a.lr),
                               __fadd_rn(__fsqrt_rn(__fdiv_rn(s[1], __fsub_rn(1.f, a.p2))), a.eps));
    s[2] = __fsub_rn(__fadd_rn(__fmul_rn(a.beta1, s[2]), __fmul_rn(__fsub_rn(1.f, a.beta1), gi)),
                     __fmul_rn(__fsub_rn(dt, __fmul_rn(a.beta1, s[0])), w));
    s[0] = dt;
    return __fdiv_rn(-s[2], dt);
  }
  if (OP == kUpdAdaGrad) {
    // AdagradDnsRspDnsKernel<cpu> (2507-2531), state history; wd is refused on the host
    float gr = __fmul_rn(g, a.rescale);
    if (a.clip >= 0.f) gr = clipf(gr, a.clip);
    s[0] = __fadd_rn(s[0], __fmul_rn(gr, gr));
    return __fsub_rn(w, __fmul_rn(__fdiv_rn(gr, __fsqrt_rn(__fadd_rn(s[0], a.eps))), a.lr));
  }
  // FtrlUpdateKernel (2133-2158), states z, n: z is updated before n; the result is MULTIPLIED by
  // gt(|z|, lamda1), so it is -0.0 for -lamda1 < z < 0 and NaN when the quotient is infinite.
  // FtrlDnsRspDnsKernel (2186-2219), the row_sparse form, computes the same tree per element.
  float gr = __fmul_rn(g, a.rescale);
  if (a.clip >= 0.f) gr = clipf(gr, a.clip);
  const float g2 = __fmul_rn(gr, gr);
  s[0] = __fadd_rn(s[0], __fsub_rn(gr, __fdiv_rn(__fmul_rn(__fsub_rn(__fsqrt_rn(__fadd_rn(s[1], g2)),
                                                                    __fsqrt_rn(s[1])), w), a.lr)));
  s[1] = __fadd_rn(s[1], g2);
  const float z = s[0];
  const float sgn = z < 0.f ? -1.f : (z > 0.f ? 1.f : 0.f);  // mshadow_op::sign
  return __fmul_rn(__fdiv_rn(__fsub_rn(__fmul_rn(sgn, a.lamda1), z),
                             __fadd_rn(__fdiv_rn(__fadd_rn(a.beta, __fsqrt_rn(s[1])), a.lr), a.wd)),
                   fabsf(z) > a.lamda1 ? 1.f : 0.f);
}

}  // namespace b200kv
