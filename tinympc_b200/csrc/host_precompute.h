// host_precompute.h — one-time cache precompute on the host (product code).
//
// Restates tiny_precompute_and_set_cache (TinyMPC src/tinympc/tiny_api.cpp:307-381):
//   Q1 = diag(Q) + rho I, R1 = diag(R) + rho I            (:317-318; Q,R already hold +rho once: "double rho")
//   P <- rho I, K_prev <- 0                                (:330-333)
//   repeat <= 1000:  K = (R1 + B'PB)^-1 B'PA ;  Pn = Q1 + A'P(A - BK) ; stop if max|K - K_prev| < 1e-5   (:335-349)
//   Quu_inv = (R1 + B'Pinf B)^-1 ; AmBKt = (A - B Kinf)' ; APf = AmBKt Pinf f ; BPf = B' Pinf f   (:352-357)
// The result agrees with Eigen's to rounding (different summation order / LU), not bit-for-bit; the solve
// kernels accept ANY cache through the C ABI, so parity of the solve path never depends on this routine.
#pragma once
#include <cmath>
#include <vector>

namespace tmpc {

template <typename T>
struct Mat {  // column-major
    int r, c;
    std::vector<T> a;
    Mat(int r_, int c_) : r(r_), c(c_), a((size_t)r_ * c_, T(0)) {}
    T &operator()(int i, int j) { return a[i + (size_t)j * r]; }
    T operator()(int i, int j) const { return a[i + (size_t)j * r]; }
};

template <typename T>
Mat<T> mul(const Mat<T> &X, const Mat<T> &Y) {
    Mat<T> Z(X.r, Y.c);
    for (int j = 0; j < Y.c; ++j)
        for (int l = 0; l < X.c; ++l) {
            const T y = Y(l, j);
            for (int i = 0; i < X.r; ++i) Z(i, j) += X(i, l) * y;
        }
    return Z;
}
template <typename T>
Mat<T> tr(const Mat<T> &X) {
    Mat<T> Z(X.c, X.r);
    for (int j = 0; j < X.c; ++j)
        for (int i = 0; i < X.r; ++i) Z(j, i) = X(i, j);
    return Z;
}
template <typename T>
Mat<T> sub(const Mat<T> &X, const Mat<T> &Y) {
    Mat<T> Z(X.r, X.c);
    for (size_t e = 0; e < Z.a.size(); ++e) Z.a[e] = X.a[e] - Y.a[e];
    return Z;
}
template <typename T>
Mat<T> add(const Mat<T> &X, const Mat<T> &Y) {
    Mat<T> Z(X.r, X.c);
    for (size_t e = 0; e < Z.a.size(); ++e) Z.a[e] = X.a[e] + Y.a[e];
    return Z;
}

// Gauss-Jordan with partial pivoting; returns false when singular
template <typename T>
bool invert(const Mat<T> &Xin, Mat<T> &inv) {
    const int n = Xin.r;
    Mat<T> X = Xin;
    inv = Mat<T>(n, n);
    for (int i = 0; i < n; ++i) inv(i, i) = T(1);
    for (int c = 0; c < n; ++c) {
        int piv = c;
        for (int i = c + 1; i < n; ++i)
            if (std::fabs(X(i, c)) > std::fabs(X(piv, c))) piv = i;
        if (X(piv, c) == T(0)) return false;
        if (piv != c)
            for (int j = 0; j < n; ++j) {
                std::swap(X(c, j), X(piv, j));
                std::swap(inv(c, j), inv(piv, j));
            }
        const T d = T(1) / X(c, c);
        for (int j = 0; j < n; ++j) {
            X(c, j) *= d;
            inv(c, j) *= d;
        }
        for (int i = 0; i < n; ++i) {
            if (i == c) continue;
            const T m = X(i, c);
            if (m == T(0)) continue;
            for (int j = 0; j < n; ++j) {
                X(i, j) -= m * X(c, j);
                inv(i, j) -= m * inv(c, j);
            }
        }
    }
    return true;
}

template <typename T>
int precompute_cache(int nx, int nu, double rho_d, const T *Ap, const T *Bp, const T *fp, const T *Q, const T *R,
                     T *Kinf_o, T *Pinf_o, T *Quu_o, T *AmBKt_o, T *APf_o, T *BPf_o) {
    const T rho = (T)rho_d;
    Mat<T> A(nx, nx), B(nx, nu), f(nx, 1), Q1(nx, nx), R1(nu, nu), P(nx, nx), Kprev(nu, nx), K(nu, nx), Pn(nx, nx);
    A.a.assign(Ap, Ap + (size_t)nx * nx);
    B.a.assign(Bp, Bp + (size_t)nx * nu);
    f.a.assign(fp, fp + nx);
    for (int i = 0; i < nx; ++i) {
        Q1(i, i) = Q[i] + rho;
        P(i, i) = rho;
    }
    for (int j = 0; j < nu; ++j) R1(j, j) = R[j] + rho;
    const Mat<T> Bt = tr(B), At = tr(A);
    int sweeps = 0;
    for (int it = 0; it < 1000; ++it) {
        const Mat<T> BtP = mul(Bt, P);
        Mat<T> Sinv(nu, nu);
        if (!invert(add(R1, mul(BtP, B)), Sinv)) return -1;
        K = mul(Sinv, mul(BtP, A));
        Pn = add(Q1, mul(mul(At, P), sub(A, mul(B, K))));
        sweeps = it + 1;
        T md = T(0);
        for (size_t e = 0; e < K.a.size(); ++e) md = std::max(md, (T)std::fabs(K.a[e] - Kprev.a[e]));
        if (md < (T)1e-5) break;
        Kprev = K;
        P = Pn;
    }
    Mat<T> Quu(nu, nu);
    if (!invert(add(R1, mul(mul(Bt, Pn), B)), Quu)) return -1;
    const Mat<T> AmBKt = tr(sub(A, mul(B, K)));
    const Mat<T> Pf = mul(Pn, f);
    const Mat<T> APf = mul(AmBKt, Pf), BPf = mul(Bt, Pf);
    std::copy(K.a.begin(), K.a.end(), Kinf_o);
    std::copy(Pn.a.begin(), Pn.a.end(), Pinf_o);
    std::copy(Quu.a.begin(), Quu.a.end(), Quu_o);
    std::copy(AmBKt.a.begin(), AmBKt.a.end(), AmBKt_o);
    std::copy(APf.a.begin(), APf.a.end(), APf_o);
    std::copy(BPf.a.begin(), BPf.a.end(), BPf_o);
    return sweeps;
}

// Sensitivity tables dKinf/drho (nu x nx) and dPinf/drho (nx x nx) of one model: the forward-mode derivative, with respect
// to rho, of the batched precompute as it runs (tinympc_b200_precompute_cache_batch: Q = Qdiag + rho, R = Rdiag + rho, then
// precompute_cache above), tangent carried next to the same primal recursion and ended by the primal's own stop test:
//   dQ1 = dR1 = 2 I (rho enters Q1, R1 twice), dP = I (P starts at rho I)
//   per sweep, S = R1 + B'PB:  dS = dR1 + B'dP B ;  dK = S^-1 (B'dP A - dS K) ;  dPn = (dQ1 + A'dP (A - BK)) - A'P (B dK)
// (the role rho_benchmark.cpp:215-229's tables play for the reference's one hard-coded quadrotor).  Q, R here are the
// USER's diagonals, without rho.  Returns the sweeps used, or -1 exactly when precompute_cache would.
template <typename T>
int precompute_sensitivity(int nx, int nu, T rho, const T *Ap, const T *Bp, const T *Q, const T *R, T *dK_o, T *dP_o) {
    Mat<T> A(nx, nx), B(nx, nu), Q1(nx, nx), R1(nu, nu), dR1(nu, nu), P(nx, nx), Kprev(nu, nx), K(nu, nx), Pn(nx, nx);
    Mat<T> dP(nx, nx), dK(nu, nx), dPn(nx, nx);
    A.a.assign(Ap, Ap + (size_t)nx * nx);
    B.a.assign(Bp, Bp + (size_t)nx * nu);
    for (int i = 0; i < nx; ++i) {
        Q1(i, i) = (Q[i] + rho) + rho;
        P(i, i) = rho;
        dP(i, i) = T(1);
    }
    for (int j = 0; j < nu; ++j) {
        R1(j, j) = (R[j] + rho) + rho;
        dR1(j, j) = T(2);
    }
    const Mat<T> Bt = tr(B), At = tr(A);
    for (int it = 0;; ++it) {
        const Mat<T> BtP = mul(Bt, P), dBtP = mul(Bt, dP);
        Mat<T> Sinv(nu, nu);
        if (!invert(add(R1, mul(BtP, B)), Sinv)) return -1;
        K = mul(Sinv, mul(BtP, A));
        dK = mul(Sinv, sub(mul(dBtP, A), mul(add(dR1, mul(dBtP, B)), K)));
        const Mat<T> AmBK = sub(A, mul(B, K)), AtP = mul(At, P);
        Pn = add(Q1, mul(AtP, AmBK));
        dPn = mul(mul(At, dP), AmBK);
        for (int i = 0; i < nx; ++i) dPn(i, i) = T(2) + dPn(i, i);
        dPn = sub(dPn, mul(AtP, mul(B, dK)));
        T md = T(0);
        for (size_t e = 0; e < K.a.size(); ++e) md = std::max(md, (T)std::fabs(K.a[e] - Kprev.a[e]));
        if (md < (T)1e-5 || it == 999) {
            Mat<T> Quu(nu, nu);
            if (!invert(add(R1, mul(mul(Bt, Pn), B)), Quu)) return -1;
            std::copy(dK.a.begin(), dK.a.end(), dK_o);
            std::copy(dPn.a.begin(), dPn.a.end(), dP_o);
            return it + 1;
        }
        Kprev = K;
        P = Pn;
        dP = dPn;
    }
}

}  // namespace tmpc
