// gpk_es.cuh — expectation propagation for p_min, the distribution of the minimiser over Nb representer points
// (robo/util/epmgp.py: joint_min, min_faktor, lt_factor, log_relative_gauss), and the entropy change of the
// candidates (robo/acquisition_functions/information_gain.py), the two device halves of entropy search.
//
// gpk_ep_kernel: one CTA per representer point k runs the EP problem of k.  V (Nb x Nb), M and the messages P, MP and
// logS live in shared memory; each lt_factor step is one rank-1 update of V.  Every elementwise step of the sweep is
// rounded explicitly in the reference's order (__dmul_rn / __dadd_rn / __ddiv_rn: no fma contraction), so the sweep
// counts equal the numpy restatement's (tests/es_model.py).  The closed form for logZ and its derivatives follows,
// solving the (Nb-1)^2 SPD system IRSR = I + R^T Sigma R by a Cholesky factor in the CTA.
// gpk_ep_norm_kernel + gpk_ep_apply_kernel: the renormalisation at the end of joint_min.
//
// Quirks of the reference kept on purpose:
//   - eps in the message clamps is the float32 epsilon (epmgp.py:7), not DBL_EPSILON;
//   - joint_min's Zij = Zm.T * Zm is, for the 1-D Zm, the elementwise square broadcast along the rows, not an outer
//     product: adds[i][j] = -gg[i][j] + Zm[j]^2;
//   - dlogZdSigma of one problem is symmetrised with a halved diagonal, 0.5 (X + X^T - diag X), and packed as its lower
//     triangle in row-major order (what rot90(., 2)[triu_indices][::-1] produces).
#pragma once
#include "gpk_internal.cuh"

#define GPK_EP_MAX_NB 64
#define GPK_EP_THREADS 256
#define GPK_EP_SWEEPS 50
#define GPK_EP_EPS 1.1920928955078125e-07      // numpy.finfo(numpy.float32).eps
#define GPK_EP_SQ2 1.4142135623730951           // numpy.sqrt(2)
#define GPK_EP_ISQ2 0.7071067811865475          // 1 / numpy.sqrt(2), rounded once (np.eye(D) / sq2)
#define GPK_EP_L2P 1.8378770664093453           // numpy.log(2) + numpy.log(numpy.pi)
// shared memory of gpk_ep_kernel: V (later IRSR and its factor), G = L^-1 R^T, A, and 9 vectors, each padded to 64
#define GPK_EP_SMEM ((3 * GPK_EP_MAX_NB * GPK_EP_MAX_NB + 9 * GPK_EP_MAX_NB) * 8)

// per-problem status written by gpk_ep_kernel
#define GPK_EP_OK 0
#define GPK_EP_NAN_VARIANCE 1                    // lt_factor produced a NaN variance (the reference raises Exception)
#define GPK_EP_IRSR_NOT_PD 2                     // IRSR not PD even with +1e-6 I (numpy.linalg.LinAlgError)

// numpy.max([a, b]): NaN propagates, otherwise a unless b is larger
__device__ __forceinline__ double gpk_np_max2(double a, double b) {
    return (a >= b || isnan(a)) ? a : b;
}

// IRSR = I + R^T Sigma R (+ jitter I) into S (D1 x D1).  R has two entries per column j: rho_j in row l_j and -rho_j in
// row k, so (R^T Sigma R)[a][b] = rho_a rho_b ((Sigma[la][lb] - Sigma[la][k]) - Sigma[k][lb] + Sigma[k][k]).
__device__ __forceinline__ void gpk_ep_build_irsr(const double* __restrict__ Sig, int D, int k, const double* rho,
                                                  double jitter, double* S) {
    const int D1 = D - 1;
    for (int x = threadIdx.x; x < D1 * D1; x += blockDim.x) {
        const int a = x / D1, b = x - a * D1;
        const int la = a < k ? a : a + 1, lb = b < k ? b : b + 1;
        const double q = __dadd_rn(__dsub_rn(__dsub_rn(Sig[la * D + lb], Sig[la * D + k]), Sig[k * D + lb]), Sig[k * D + k]);
        double v = __dadd_rn(a == b ? 1.0 : 0.0, __dmul_rn(__dmul_rn(rho[a], rho[b]), q));
        if (a == b) v = __dadd_rn(v, jitter);
        S[x] = v;
    }
}

// One EP problem per CTA (blockIdx.x = k).  mu (D), Sig (D x D) the posterior at the representer points.  Writes the
// un-normalised logZ[k], dMu[k][D], dMuMu[k][D][D], dSig[k][D (D + 1) / 2], sweeps[k] and status[k].
__global__ void __launch_bounds__(GPK_EP_THREADS) gpk_ep_kernel(const double* __restrict__ mu, const double* __restrict__ Sig,
                                                                 int D, double* __restrict__ logZ, double* __restrict__ dMu,
                                                                 double* __restrict__ dMuMu, double* __restrict__ dSig,
                                                                 int* __restrict__ sweeps, int* __restrict__ status)
{
    extern __shared__ double es_sm[];
    double* V = es_sm;                                        // D x D working covariance; then IRSR / its factor
    double* G = V + GPK_EP_MAX_NB * GPK_EP_MAX_NB;            // (D - 1) x D: L^-1 R^T
    double* A = G + GPK_EP_MAX_NB * GPK_EP_MAX_NB;            // D x D: R IRSR^-1 R^T
    double* M = A + GPK_EP_MAX_NB * GPK_EP_MAX_NB;
    double* Vc = M + GPK_EP_MAX_NB;                           // (V[:, l] - V[:, k]) / sq2; later rho
    double* Pm = Vc + GPK_EP_MAX_NB;
    double* MP = Pm + GPK_EP_MAX_NB;
    double* logS = MP + GPK_EP_MAX_NB;
    double* r = logS + GPK_EP_MAX_NB;
    double* b = r + GPK_EP_MAX_NB;
    double* Ab = b + GPK_EP_MAX_NB;
    double* Sr = Ab + GPK_EP_MAX_NB;
    __shared__ int s_nan;
    __shared__ int s_fail;
    __shared__ double s_rk;

    const int k = blockIdx.x, t = threadIdx.x, D1 = D - 1, T = D * (D + 1) / 2;
    for (int x = t; x < D * D; x += blockDim.x) V[x] = Sig[x];
    for (int x = t; x < D; x += blockDim.x) {
        M[x] = mu[x];
        Pm[x] = 0.0;
        MP[x] = 0.0;
        logS[x] = 0.0;
    }
    if (t == 0) s_nan = 0;
    __syncthreads();

    // ---- sweeps (min_faktor / lt_factor with gamma = 1) ----
    int sw = 0;
    double d = 0.0;
    for (int count = 0; count < GPK_EP_SWEEPS; ++count) {
        ++sw;
        double diff = 0.0;
        for (int i = 0; i < D1; ++i) {
            const int l = i < k ? i : i + 1;
            const double p = Pm[i], mp = MP[i];
            const double cVc = __ddiv_rn(__dadd_rn(__dsub_rn(V[l * D + l], __dmul_rn(2.0, V[k * D + l])), V[k * D + k]), 2.0);
            const double cM = __ddiv_rn(__dsub_rn(M[l], M[k]), GPK_EP_SQ2);
            const double cVnic = gpk_np_max2(__ddiv_rn(cVc, __dsub_rn(1.0, __dmul_rn(p, cVc))), 0.0);
            const double cmni = __dadd_rn(cM, __dmul_rn(cVnic, __dsub_rn(__dmul_rn(p, cM), mp)));
            double z = __ddiv_rn(cmni, __dsqrt_rn(__dadd_rn(cVnic, 1e-25)));
            if (isnan(z)) z = -INFINITY;
            const int exit_flag = z < -6.0 ? -1 : (z > 6.0 ? 1 : 0);
            double pnew = 0.0, mpnew = 0.0, lS = 0.0, dp, dmp;
            if (exit_flag == 0) {
                const double logphi = __dmul_rn(-0.5, __dadd_rn(__dmul_rn(z, z), GPK_EP_L2P));
                const double lP = log(__dmul_rn(0.5, erfc(__ddiv_rn(-z, GPK_EP_SQ2))));
                const double e = exp(__dsub_rn(logphi, lP));
                const double alpha = __ddiv_rn(e, __dsqrt_rn(cVnic));
                const double beta = __dmul_rn(alpha, __dadd_rn(__dmul_rn(alpha, cVnic), cmni));
                const double rr = __ddiv_rn(beta, __dsub_rn(1.0, beta));
                pnew = __ddiv_rn(rr, cVnic);
                mpnew = __dadd_rn(__dmul_rn(rr, __dadd_rn(alpha, __ddiv_rn(cmni, cVnic))), alpha);
                dp = gpk_np_max2(__dadd_rn(-p, GPK_EP_EPS), __dsub_rn(pnew, p));
                dmp = gpk_np_max2(__dadd_rn(-mp, GPK_EP_EPS), __dsub_rn(mpnew, mp));
                d = gpk_np_max2(dmp, dp);
                pnew = __dadd_rn(p, dp);
                mpnew = __dadd_rn(mp, dmp);
                lS = __dadd_rn(__dsub_rn(lP, __dmul_rn(0.5, __dsub_rn(__dsub_rn(log(beta), log(pnew)), log(cVnic)))),
                               __dmul_rn(__ddiv_rn(__dmul_rn(alpha, alpha), __dmul_rn(2.0, beta)), cVnic));
            } else if (exit_flag == 1) {
                dp = -p;
                dmp = -mp;
                d = dp > dmp ? dp : dmp;                      // Python's max([dmp, dp])
            } else {
                d = NAN;
            }
            __syncthreads();                                  // every thread has read P[i], MP[i], M, V
            if (exit_flag == -1) break;                       // the problem ends with logZ = -inf (below)
            if (t < D) Vc[t] = __ddiv_rn(__dsub_rn(V[t * D + l], V[t * D + k]), GPK_EP_SQ2);
            if (t == 0) {
                Pm[i] = pnew;
                MP[i] = mpnew;
                logS[i] = lS;
            }
            __syncthreads();
            const double den = __dadd_rn(1.0, __dmul_rn(dp, cVc));
            const double cv = __ddiv_rn(dp, den);
            const double cm = __ddiv_rn(__dsub_rn(dmp, __dmul_rn(cM, dp)), den);
            for (int x = t; x < D * D; x += blockDim.x) {
                const int a = x / D, c = x - a * D;
                const double v = __dsub_rn(V[x], __dmul_rn(cv, __dmul_rn(Vc[a], Vc[c])));
                if (isnan(v)) s_nan = 1;
                V[x] = v;
            }
            if (t < D) M[t] = __dadd_rn(M[t], __dmul_rn(cm, Vc[t]));
            __syncthreads();
            if (exit_flag == 0 && s_nan) {
                if (t == 0) status[k] = GPK_EP_NAN_VARIANCE;
                return;
            }
            if (isnan(d)) break;
            diff = __dadd_rn(diff, fabs(d));
        }
        if (isnan(d)) break;
        if (fabs(diff) < 0.001) break;
    }

    double* outMu = dMu + (size_t)k * D;
    double* outMuMu = dMuMu + (size_t)k * D * D;
    double* outSig = dSig + (size_t)k * T;
    if (t == 0) sweeps[k] = sw;
    if (isnan(d)) {
        if (t == 0) {
            logZ[k] = -INFINITY;
            status[k] = GPK_EP_OK;
        }
        for (int x = t; x < D; x += blockDim.x) outMu[x] = 0.0;
        for (int x = t; x < D * D; x += blockDim.x) outMuMu[x] = 0.0;
        for (int x = t; x < T; x += blockDim.x) outSig[x] = 0.0;
        return;
    }

    // ---- closed form for logZ and its derivatives ----
    double* rho = Vc;
    if (t < D1) rho[t] = __dmul_rn(__dsqrt_rn(Pm[t]), GPK_EP_ISQ2);
    if (t == 0) {
        double rk = 0.0;
        for (int j = 0; j < D1; ++j) rk = __dadd_rn(rk, __dmul_rn(MP[j], -GPK_EP_ISQ2));
        s_rk = rk;
    }
    __syncthreads();
    if (t < D) {
        const int j = t < k ? t : t - 1;                      // column of C whose row l_j is t
        r[t] = t == k ? s_rk : __dmul_rn(MP[j], GPK_EP_ISQ2);
    }
    // Cholesky of IRSR in place (left-looking), retried with +1e-10 I and +1e-6 I (epmgp.py:147-153)
    double* L = V;
    bool pd = false;
    for (int attempt = 0; attempt < 3 && !pd; ++attempt) {
        gpk_ep_build_irsr(Sig, D, k, rho, attempt == 0 ? 0.0 : (attempt == 1 ? 1e-10 : 1e-6), L);
        if (t == 0) s_fail = 0;
        __syncthreads();
        for (int j = 0; j < D1; ++j) {
            if (t == 0) {
                double s = L[j * D1 + j];
                for (int m = 0; m < j; ++m) s = __dsub_rn(s, __dmul_rn(L[j * D1 + m], L[j * D1 + m]));
                if (!(s > 0.0)) s_fail = 1;
                L[j * D1 + j] = __dsqrt_rn(s);
            }
            __syncthreads();
            if (s_fail) break;
            const double ljj = L[j * D1 + j];
            for (int i2 = j + 1 + t; i2 < D1; i2 += blockDim.x) {
                double s = L[i2 * D1 + j];
                for (int m = 0; m < j; ++m) s = __dsub_rn(s, __dmul_rn(L[i2 * D1 + m], L[j * D1 + m]));
                L[i2 * D1 + j] = __ddiv_rn(s, ljj);
            }
            __syncthreads();
        }
        pd = !s_fail;
        __syncthreads();
    }
    if (!pd) {
        if (t == 0) status[k] = GPK_EP_IRSR_NOT_PD;
        return;
    }
    // G = L^-1 R^T, one column per thread: R^T[j][c] = rho_j if c == l_j, -rho_j if c == k
    if (t < D) {
        const int c = t;
        for (int j = 0; j < D1; ++j) {
            const int lj = j < k ? j : j + 1;
            double s = c == lj ? rho[j] : (c == k ? -rho[j] : 0.0);
            for (int m = 0; m < j; ++m) s = __dsub_rn(s, __dmul_rn(L[j * D1 + m], G[m * D + c]));
            G[j * D + c] = __ddiv_rn(s, L[j * D1 + j]);
        }
    }
    __syncthreads();
    for (int x = t; x < D * D; x += blockDim.x) {             // A = G^T G (exactly symmetric)
        const int a = x / D, c = x - a * D;
        double s = 0.0;
        for (int m = 0; m < D1; ++m) s = __dadd_rn(s, __dmul_rn(G[m * D + a], G[m * D + c]));
        A[x] = s;
    }
    if (t < D) {                                              // Sr = Sigma r, b = Mu + Sigma r
        double s = 0.0;
        for (int j = 0; j < D; ++j) s = __dadd_rn(s, __dmul_rn(Sig[t * D + j], r[j]));
        Sr[t] = s;
        b[t] = __dadd_rn(mu[t], s);
    }
    __syncthreads();
    if (t < D) {                                              // Ab = A b (= b^T A: A is symmetric)
        double s = 0.0;
        for (int j = 0; j < D; ++j) s = __dadd_rn(s, __dmul_rn(A[t * D + j], b[j]));
        Ab[t] = s;
    }
    __syncthreads();
    if (t == 0) {
        double rSr = 0.0, bAb = 0.0, Mur = 0.0, dts = 0.0, s = 0.0, mpm = 0.0;
        for (int j = 0; j < D; ++j) {
            rSr = __dadd_rn(rSr, __dmul_rn(r[j], Sr[j]));
            bAb = __dadd_rn(bAb, __dmul_rn(b[j], Ab[j]));
            Mur = __dadd_rn(Mur, __dmul_rn(mu[j], r[j]));
        }
        for (int j = 0; j < D1; ++j) {
            dts = __dadd_rn(dts, log(L[j * D1 + j]));
            s = __dadd_rn(s, logS[j]);
            if (MP[j] != 0.0) mpm = __dadd_rn(mpm, __ddiv_rn(__dmul_rn(MP[j], MP[j]), Pm[j]));
        }
        dts = __dmul_rn(2.0, dts);
        logZ[k] = __dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(0.5, __dsub_rn(__dsub_rn(rSr, bAb), dts)), Mur), s),
                            __dmul_rn(0.5, mpm));
        status[k] = GPK_EP_OK;
    }
    for (int x = t; x < D; x += blockDim.x) outMu[x] = __dsub_rn(r[x], Ab[x]);
    for (int x = t; x < D * D; x += blockDim.x) outMuMu[x] = -A[x];
    // dlogZdSigma = -A - 2 r Ab^T + r r^T + Ab Ab^T, symmetrised with a halved diagonal, lower triangle row-major
    for (int x = t; x < D * D; x += blockDim.x) {
        const int a = x / D, c = x - a * D;
        if (c > a) continue;
        const double xac = __dadd_rn(__dadd_rn(__dsub_rn(-A[a * D + c], __dmul_rn(2.0, __dmul_rn(r[a], Ab[c]))),
                                               __dmul_rn(r[a], r[c])), __dmul_rn(Ab[a], Ab[c]));
        double v;
        if (a == c) {
            v = __dmul_rn(0.5, xac);
        } else {
            const double xca = __dadd_rn(__dadd_rn(__dsub_rn(-A[c * D + a], __dmul_rn(2.0, __dmul_rn(r[c], Ab[a]))),
                                                   __dmul_rn(r[c], r[a])), __dmul_rn(Ab[c], Ab[a]));
            v = __dmul_rn(0.5, __dadd_rn(xac, xca));
        }
        outSig[a * (a + 1) / 2 + c] = v;
    }
}

// joint_min's renormalisation (epmgp.py:54-81), one CTA: logP in place (-inf and +inf -> -500 first, then minus the
// log-sum-exp, which falls back to the max when infinite); Zm, Zs and adds = -gg + Zm^2 (see the header) for
// gpk_ep_apply_kernel.  Every sum runs over k in index order.
__global__ void __launch_bounds__(GPK_EP_THREADS) gpk_ep_norm_kernel(int D, double* __restrict__ logP,
                                                                      const double* __restrict__ dMu,
                                                                      const double* __restrict__ dMuMu,
                                                                      const double* __restrict__ dSig,
                                                                      double* __restrict__ Zm, double* __restrict__ Zs,
                                                                      double* __restrict__ adds)
{
    __shared__ double e[GPK_EP_MAX_NB], zm[GPK_EP_MAX_NB], lp[GPK_EP_MAX_NB];
    __shared__ double sZ, sS;
    const int t = threadIdx.x, T = D * (D + 1) / 2;
    if (t < D) {
        const double v = logP[t];
        lp[t] = isinf(v) ? -500.0 : v;
        e[t] = exp(lp[t]);
    }
    __syncthreads();
    if (t == 0) {
        double Z = 0.0, mx = lp[0];
        for (int k = 0; k < D; ++k) Z = __dadd_rn(Z, e[k]);
        for (int k = 1; k < D; ++k) mx = gpk_np_max2(mx, lp[k]);
        double s = 0.0;
        for (int k = 0; k < D; ++k) s = __dadd_rn(s, exp(__dsub_rn(lp[k], mx)));
        s = __dadd_rn(mx, log(s));
        sS = isinf(s) ? mx : s;
        sZ = Z;
    }
    __syncthreads();
    const double Z = sZ;
    if (t < D) {
        logP[t] = __dsub_rn(lp[t], sS);
        double s = 0.0;
        for (int k = 0; k < D; ++k) s = __dadd_rn(s, __dmul_rn(e[k], dMu[k * D + t]));
        zm[t] = __ddiv_rn(s, Z);
        Zm[t] = zm[t];
    }
    for (int x = t; x < T; x += blockDim.x) {
        double s = 0.0;
        for (int k = 0; k < D; ++k) s = __dadd_rn(s, __dmul_rn(e[k], dSig[(size_t)k * T + x]));
        Zs[x] = __ddiv_rn(s, Z);
    }
    __syncthreads();
    for (int x = t; x < D * D; x += blockDim.x) {
        const int i = x / D, j = x - i * D;
        double s = 0.0;
        for (int k = 0; k < D; ++k) {
            const double f = __dadd_rn(dMuMu[(size_t)k * D * D + x], __dmul_rn(dMu[k * D + i], dMu[k * D + j]));
            s = __dadd_rn(s, __dmul_rn(f, e[k]));
        }
        adds[x] = __dadd_rn(-__ddiv_rn(s, Z), __dmul_rn(zm[j], zm[j]));
    }
}

// one CTA per problem k: dlogPdMu[k] -= Zm, dlogPdSigma[k] -= Zs, dlogPdMudMu[k] += adds
__global__ void gpk_ep_apply_kernel(int D, double* __restrict__ dMu, double* __restrict__ dMuMu, double* __restrict__ dSig,
                                    const double* __restrict__ Zm, const double* __restrict__ Zs,
                                    const double* __restrict__ adds)
{
    const int k = blockIdx.x, T = D * (D + 1) / 2;
    for (int x = threadIdx.x; x < D; x += blockDim.x) dMu[k * D + x] = __dsub_rn(dMu[k * D + x], Zm[x]);
    for (int x = threadIdx.x; x < T; x += blockDim.x) dSig[(size_t)k * T + x] = __dsub_rn(dSig[(size_t)k * T + x], Zs[x]);
    for (int x = threadIdx.x; x < D * D; x += blockDim.x)
        dMuMu[(size_t)k * D * D + x] = __dadd_rn(dMuMu[(size_t)k * D * D + x], adds[x]);
}

// ---------------------------------------------------------------------------------------------------------------------
// The entropy change of one candidate (InformationGain._dh_fun, robo/acquisition_functions/information_gain.py:169-203)
// given its predictive variance v and its covariance sigma (Nb) to the representer points.
//
// Cross-covariance: sigma_j = (k(zb_j, x) - K(x, X) U[:, j]) * y_std^2 (output transform), clipped at DBL_EPSILON like
// every entry of predict(full_cov=True) (gaussian_process.py:290-294), U = K^-1 K(X, zb) (N x Nb) built once per update.

#define GPK_ES_THREADS 256

// k(a, b) of the handle's kernel on scaled inputs: amp * prod_g f(sum_{t in g} (a - b)^2 / metric_t), times the
// kernel's factor when it has one
__device__ __forceinline__ double gpk_es_kval(const KSpec& s, const double* a, const double* b) {
    double prod = 1.0, r2 = 0.0;
    for (int t = 0; t < s.n_terms; ++t) {
        const double dd = a[s.axis[t]] - b[s.axis[t]];
        r2 += dd * dd * s.inv_metric[t];
        if (s.last[t]) {
            prod *= gpk_radial(s.family, r2);
            r2 = 0.0;
        }
    }
    const double k = s.amp * prod;
    return s.factor.kind != GPK_FACTOR_NONE ? k * gpk_factor_value(s.factor, a[s.factor.axis], b[s.factor.axis]) : k;
}

// raw representer points -> scaled (x - lower) / (upper - lower) when the handle scales its inputs
__global__ void gpk_es_scale_kernel(const double* __restrict__ Z, int nb, int d, const double* __restrict__ lo,
                                    const double* __restrict__ up, double* __restrict__ Zs) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nb * d) return;
    const int a = t % d;
    double v = Z[t];
    if (lo != nullptr) v = (v - lo[a]) / (up[a] - lo[a]);
    Zs[t] = v;
}

// Kxz[n][j] = k(X_n, zb_j) for the n training rows (rows n .. NP-1 stay zero)
__global__ void gpk_es_kxz_kernel(KSpec s, const double* __restrict__ X, int n, int d, const double* __restrict__ Zs,
                                  int nb, double* __restrict__ Kxz) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long)n * nb) return;
    const int i = (int)(t / nb), j = (int)(t - (long)i * nb);
    Kxz[t] = gpk_es_kval(s, X + (size_t)i * d, Zs + (size_t)j * d);
}

// B = P A (lower P, NP x NP row-major) or B = P^T A (trans = 1); A, B are NP x nb.  One thread per entry, index order.
__global__ void gpk_es_trmm_kernel(const double* __restrict__ P, int NP, const double* __restrict__ A, int nb, int trans,
                                   double* __restrict__ B) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long)NP * nb) return;
    const int r = (int)(t / nb), j = (int)(t - (long)r * nb);
    double s = 0.0;
    if (!trans)
        for (int c = 0; c <= r; ++c) s = fma(P[(size_t)r * NP + c], A[(size_t)c * nb + j], s);
    else
        for (int c = r; c < NP; ++c) s = fma(P[(size_t)c * NP + r], A[(size_t)c * nb + j], s);
    B[t] = s;
}

// one CTA per candidate: sigma (rows x nb).  K(x, X) in tiles of GPK_ES_THREADS training rows through shared memory,
// thread j < nb accumulates sum_n k(x, X_n) U[n][j] in index order.  The fp64 K* is never stored in HBM.
__global__ void __launch_bounds__(GPK_ES_THREADS) gpk_es_sigma_kernel(KSpec s, const double* __restrict__ Xs, long rows,
                                                                      int d, const double* __restrict__ lo,
                                                                      const double* __restrict__ up,
                                                                      const double* __restrict__ X, int n,
                                                                      const double* __restrict__ U,
                                                                      const double* __restrict__ Zs, int nb,
                                                                      double out_scale, double* __restrict__ sig) {
    __shared__ double xs[GPK_MAX_TERMS];
    __shared__ double ks[GPK_ES_THREADS];
    const long c = blockIdx.x;
    const int t = threadIdx.x;
    if (t < d) {
        double v = Xs[c * d + t];
        if (lo != nullptr) v = (v - lo[t]) / (up[t] - lo[t]);
        xs[t] = v;
    }
    __syncthreads();
    double acc = 0.0;
    for (int n0 = 0; n0 < n; n0 += GPK_ES_THREADS) {
        if (n0 + t < n) ks[t] = gpk_es_kval(s, xs, X + (size_t)(n0 + t) * d);
        __syncthreads();
        if (t < nb) {
            const int cnt = min(GPK_ES_THREADS, n - n0);
            for (int q = 0; q < cnt; ++q) acc = fma(ks[q], U[(size_t)(n0 + q) * nb + t], acc);
        }
        __syncthreads();
    }
    if (t < nb) {
        const double v = (gpk_es_kval(s, xs, Zs + (size_t)t * d) - acc) * out_scale;
        sig[c * nb + t] = v < GPK_EPS ? GPK_EPS : v;          // numpy.clip(cov, eps, inf): NaN stays NaN
    }
}

// One CTA per candidate: dH (information_gain.py:169-203 with the replacements of compute, :112-125).
// With iv = 1 / (v - sn2) (v_ = v - sn2 is negative where v < sn2, as in the reference) and sq = sqrt(v + 1e-10):
//   dm_a = (sigma_a iv) sq,  dv_ab = -(sigma_a iv) sigma_b (a >= b, packed lower triangle, row-major),
//   det_i = dSig[i] . dv + 0.5 (Hs[i] . dm dm^T), Hs = dlogPdMudMu[i] folded to its lower triangle (only the symmetric
//   part of the quadratic form counts), g_i = dMu[i] . dm,
//   lPred[i][p] = (logP_i + det_i) + g_i W_p, normalised per column by its log-sum-exp, or by its max in EVERY column
//   when any column's log-sum-exp is infinite (:193-195),
//   dH = mean_p (sum_i exp(lPred) (lPred + lmb_i) + H),  H = -sum_i exp(logP_i) (logP_i + lmb_i).
// Outside [lower, upper]: DBL_EPSILON (np.spacing(1), :219-222); NaN or +inf: -DBL_MAX (:119-120); -inf stays.
// The warp sums over the packed triangle end in a fixed shuffle tree; the column sum in a fixed pairwise tree.
__global__ void __launch_bounds__(GPK_ES_THREADS) gpk_es_dh_kernel(const double* __restrict__ Xs, long rows, int d,
                                                                   const double* __restrict__ blo,
                                                                   const double* __restrict__ bup,
                                                                   const double* __restrict__ var,
                                                                   const double* __restrict__ sig, int nb, int np_,
                                                                   double sn2, double H,
                                                                   const double* __restrict__ logP,
                                                                   const double* __restrict__ lmb,
                                                                   const double* __restrict__ dMu,
                                                                   const double* __restrict__ dSig,
                                                                   const double* __restrict__ Hs,
                                                                   const double* __restrict__ W,
                                                                   double* __restrict__ out) {
    __shared__ double dm[GPK_EP_MAX_NB], base[GPK_EP_MAX_NB], g[GPK_EP_MAX_NB], lm[GPK_EP_MAX_NB];
    __shared__ double dv[GPK_EP_MAX_NB * (GPK_EP_MAX_NB + 1) / 2], dmm[GPK_EP_MAX_NB * (GPK_EP_MAX_NB + 1) / 2];
    __shared__ double red[GPK_ES_THREADS];
    __shared__ int s_oob, s_inf;
    const long c = blockIdx.x;
    const int t = threadIdx.x, T = nb * (nb + 1) / 2;
    if (t == 0) { s_oob = 0; s_inf = 0; }
    __syncthreads();
    if (t < d) {
        const double x = Xs[c * d + t];
        if (x < blo[t] || x > bup[t]) s_oob = 1;
    }
    __syncthreads();
    if (s_oob) {
        if (t == 0) out[c] = GPK_EPS;
        return;
    }
    const double v = var[c];
    const double iv = 1.0 / (v - sn2);
    const double sq = sqrt(v + 1e-10);
    if (t < nb) {
        dm[t] = (sig[c * nb + t] * iv) * sq;
        lm[t] = lmb[t];
    }
    for (int x = t; x < T; x += blockDim.x) {
        int a = (int)((sqrt(8.0 * x + 1.0) - 1.0) * 0.5);
        if ((a + 1) * (a + 2) / 2 <= x) ++a;
        if (a * (a + 1) / 2 > x) --a;
        const int b = x - a * (a + 1) / 2;
        const double sa = sig[c * nb + a] * iv;
        dv[x] = -(sa * sig[c * nb + b]);
        dmm[x] = ((sig[c * nb + a] * iv) * sq) * ((sig[c * nb + b] * iv) * sq);
    }
    __syncthreads();
    const int warp = t >> 5, lane = t & 31;
    for (int i = warp; i < nb; i += GPK_ES_THREADS / 32) {
        double sd = 0.0, sh = 0.0, sg = 0.0;
        for (int x = lane; x < T; x += 32) {
            sd = fma(dSig[(size_t)i * T + x], dv[x], sd);
            sh = fma(Hs[(size_t)i * T + x], dmm[x], sh);
        }
        for (int a = lane; a < nb; a += 32) sg = fma(dMu[i * nb + a], dm[a], sg);
        for (int o = 16; o > 0; o >>= 1) {
            sd += __shfl_xor_sync(0xffffffffu, sd, o);
            sh += __shfl_xor_sync(0xffffffffu, sh, o);
            sg += __shfl_xor_sync(0xffffffffu, sg, o);
        }
        if (lane == 0) {
            base[i] = logP[i] + (sd + 0.5 * sh);
            g[i] = sg;
        }
    }
    __syncthreads();
    // pass 1: is any column's log-sum-exp infinite?
    for (int p = t; p < np_; p += blockDim.x) {
        const double w = W[p];
        double mx = base[0] + g[0] * w;
        for (int i = 1; i < nb; ++i) mx = gpk_np_max2(mx, base[i] + g[i] * w);
        double se = 0.0;
        for (int i = 0; i < nb; ++i) se += exp((base[i] + g[i] * w) - mx);
        if (isinf(mx + log(se))) s_inf = 1;
    }
    __syncthreads();
    const bool use_max = s_inf != 0;
    double acc = 0.0;
    for (int p = t; p < np_; p += blockDim.x) {
        const double w = W[p];
        double mx = base[0] + g[0] * w;
        for (int i = 1; i < nb; ++i) mx = gpk_np_max2(mx, base[i] + g[i] * w);
        double sel = mx;
        if (!use_max) {
            double se = 0.0;
            for (int i = 0; i < nb; ++i) se += exp((base[i] + g[i] * w) - mx);
            sel = mx + log(se);
        }
        double col = 0.0;
        for (int i = 0; i < nb; ++i) {
            const double l = (base[i] + g[i] * w) - sel;
            col += exp(l) * (l + lm[i]);
        }
        acc += col + H;
    }
    red[t] = acc;
    __syncthreads();
    for (int s2 = GPK_ES_THREADS / 2; s2 > 0; s2 >>= 1) {
        if (t < s2) red[t] += red[t + s2];
        __syncthreads();
    }
    if (t == 0) {
        const double dH = red[0] / (double)np_;
        out[c] = (isnan(dH) || dH == INFINITY) ? -1.7976931348623157e308 : dH;
    }
}

// ---------------------------------------------------------------------------------------
// Information gain per unit cost (robo/acquisition_functions/information_gain_per_unit_cost.py) over Fabolas models
// ---------------------------------------------------------------------------------------
// FabolasGP.normalize / MTBOGP's normalize on the device (robo/models/fabolas_gp.py:122-126, mtbo_gp.py:12-15):
// out[c][j] = (x_j - lo_j) / (up_j - lo_j) for the d - 1 configuration columns, basis(x_{d-1}) for the last (environment
// or task) column.  numpy's (1 - s) ** 2 on an array is one multiply t * t, its true division is IEEE, and CUDA's rint
// rounds half to even as np.rint does: the result is bit-identical to the host transform.
__global__ void gpk_fabolas_transform_kernel(const double* __restrict__ X, long m, int d, const double* __restrict__ lo,
                                             const double* __restrict__ up, int basis, double* __restrict__ out) {
    const long e = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m * d) return;
    const int j = (int)(e % d);
    const double x = X[e];
    double v;
    if (j < d - 1) {
        v = (x - lo[j]) / (up[j] - lo[j]);
    } else if (basis == GPK_BASIS_ONE_MINUS_S_SQ) {
        const double t = 1.0 - x;
        v = t * t;
    } else if (basis == GPK_BASIS_TASK) {
        v = rint(x);
    } else {
        v = x;
    }
    out[e] = v;
}

// out = dh / (exp(log_cost) + overhead) per model and candidate (information_gain_per_unit_cost.py:91-104) over the
// n x m values (out may be dh); -DBL_MAX / c overflows to -inf for c < 1 exactly as numpy does
__global__ void gpk_es_cost_ratio_kernel(const double* dh, const double* __restrict__ log_cost, long total,
                                         double overhead, double* out) {
    const long e = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    out[e] = dh[e] / (exp(log_cost[e]) + overhead);
}
