// bellman_b200: the BLS12-381 pairing -- Fp6 / Fp12 tower, Miller loop and final exponentiation.
//
// Stands in for what groth16::verify_proof and batch::Verifier::verify (groth16/src/verifier.rs:23-58,
// verifier/batch.rs:100-173) call in the pairing / bls12_381 crates: multi_miller_loop and
// final_exponentiation.  Tower:
//     Fp6  = Fp2[v] / (v^3 - xi),  xi = u + 1
//     Fp12 = Fp6[w] / (w^2 - v)           (so w^6 = xi: Fp12 = Fp2[w] / (w^6 - xi))
// Coefficient k of the Fp2[w] view sits at c(k % 2).c(k / 2).
//
// G_T convention: the Miller loop runs over |x| without conjugating f, and the hard part of the final
// exponentiation uses (x - 1)^2 (x + p) (x^2 + p^2 - 1) + 3 = 3 (p^4 - p^2 + 1) / r (x = -|x|), so the
// result is e(P, Q)^3 for the pairing e = f_{|x|,Q}(P)^((p^12 - 1) / r).  3 is prime to r, so "the product
// is one" is decided exactly as with e itself.  Constants come from tools/gen_constants.py.
#pragma once
#include "curve.cuh"

namespace bb {

BB_HD Fp2 fp2_mul_fp(const Fp2& a, const Fp& k) { return {a.c0 * k, a.c1 * k}; }
BB_HD Fp2 fp2_mul_xi(const Fp2& a) { return {a.c0 - a.c1, a.c0 + a.c1}; }      // (a0 + a1 u)(1 + u)
BB_HD Fp2 fp2_conj(const Fp2& a) { return {a.c0, a.c1.neg()}; }

struct Fp6 {
    Fp2 c0, c1, c2;
    BB_HD static Fp6 zero() { return {Fp2::zero(), Fp2::zero(), Fp2::zero()}; }
    BB_HD static Fp6 one() { return {fp2_one(), Fp2::zero(), Fp2::zero()}; }
    BB_HD bool is_zero() const { return c0.is_zero() && c1.is_zero() && c2.is_zero(); }
    BB_HD bool operator==(const Fp6& o) const { return c0 == o.c0 && c1 == o.c1 && c2 == o.c2; }
    BB_HD Fp6 operator+(const Fp6& o) const { return {c0 + o.c0, c1 + o.c1, c2 + o.c2}; }
    BB_HD Fp6 operator-(const Fp6& o) const { return {c0 - o.c0, c1 - o.c1, c2 - o.c2}; }
    BB_HD Fp6 neg() const { return {c0.neg(), c1.neg(), c2.neg()}; }
    BB_HD Fp6 mul_v() const { return {fp2_mul_xi(c2), c0, c1}; }               // * v, v^3 = xi
};

struct Fp12 {
    Fp6 c0, c1;
    BB_HD static Fp12 one() { return {Fp6::one(), Fp6::zero()}; }
    BB_HD bool is_one() const { return c0 == Fp6::one() && c1.is_zero(); }
    BB_HD bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
    BB_HD Fp12 conj() const { return {c0, c1.neg()}; }                           // f^(p^6); the inverse in the cyclotomic subgroup
};

// Karatsuba over Fp2: 6 Fp2 products
BB_HD_NOINLINE Fp6 fp6_mul(Fp6 a, Fp6 b) {
    Fp2 t0 = a.c0 * b.c0, t1 = a.c1 * b.c1, t2 = a.c2 * b.c2;
    Fp6 r;
    r.c0 = t0 + fp2_mul_xi((a.c1 + a.c2) * (b.c1 + b.c2) - t1 - t2);
    r.c1 = (a.c0 + a.c1) * (b.c0 + b.c1) - t0 - t1 + fp2_mul_xi(t2);
    r.c2 = (a.c0 + a.c2) * (b.c0 + b.c2) - t0 - t2 + t1;
    return r;
}
// a * (b0 + b1 v): 6 Fp2 products
BB_HD_NOINLINE Fp6 fp6_mul_01(Fp6 a, Fp2 b0, Fp2 b1) {
    return {a.c0 * b0 + fp2_mul_xi(a.c2 * b1), a.c0 * b1 + a.c1 * b0, a.c1 * b1 + a.c2 * b0};
}
// a * (b1 v): 3 Fp2 products
BB_HD Fp6 fp6_mul_1(const Fp6& a, const Fp2& b1) { return {fp2_mul_xi(a.c2 * b1), a.c0 * b1, a.c1 * b1}; }

BB_HD_NOINLINE Fp6 fp6_inv(Fp6 a) {
    Fp2 t0 = a.c0.sqr() - fp2_mul_xi(a.c1 * a.c2);
    Fp2 t1 = fp2_mul_xi(a.c2.sqr()) - a.c0 * a.c1;
    Fp2 t2 = a.c1.sqr() - a.c0 * a.c2;
    Fp2 n = a.c0 * t0 + fp2_mul_xi(a.c2 * t1 + a.c1 * t2);      // the norm down to Fp2, then fp_inv_gcd inside fp2_inv
    Fp2 ni = fp2_inv(n);
    return {t0 * ni, t1 * ni, t2 * ni};
}

// Karatsuba over Fp6: 3 Fp6 products = 18 Fp2 products
BB_HD_NOINLINE Fp12 fp12_mul(Fp12 a, Fp12 b) {
    Fp6 t0 = fp6_mul(a.c0, b.c0), t1 = fp6_mul(a.c1, b.c1);
    return {t0 + t1.mul_v(), fp6_mul(a.c0 + a.c1, b.c0 + b.c1) - t0 - t1};
}
// complex squaring: 2 Fp6 products = 12 Fp2 products
BB_HD_NOINLINE Fp12 fp12_sqr(Fp12 a) {
    Fp6 t = fp6_mul(a.c0, a.c1);
    Fp6 s = fp6_mul(a.c0 + a.c1, a.c0 + a.c1.mul_v());
    return {s - t - t.mul_v(), t + t};
}
BB_HD_NOINLINE Fp12 fp12_inv(Fp12 a) {
    Fp6 t = fp6_inv(fp6_mul(a.c0, a.c0) - fp6_mul(a.c1, a.c1).mul_v());       // (a0 + a1 w)(a0 - a1 w) = a0^2 - a1^2 v
    return {fp6_mul(a.c0, t), fp6_mul(a.c1, t).neg()};
}

// f * l for a line l = (A + B v) + (C v) w -- the shape of both Miller steps below: 15 Fp2 products
BB_HD_NOINLINE Fp12 fp12_mul_line(Fp12 f, Fp2 A, Fp2 B, Fp2 C) {
    Fp6 t0 = fp6_mul_01(f.c0, A, B);
    Fp6 t1 = fp6_mul_1(f.c1, C);
    Fp6 t2 = fp6_mul_01(f.c0 + f.c1, A, B + C);
    return {t0 + t1.mul_v(), t2 - t0 - t1};
}

// Granger-Scott squaring of an element of the cyclotomic subgroup (after the easy part of the final
// exponentiation).  View Fp12 = Fp4[w] / (w^3 - s), Fp4 = Fp2[s] / (s^2 - xi), s = w^3:
//   f = A0 + A1 w + A2 w^2 with A0 = c0.c0 + c1.c1 s, A1 = c1.c0 + c0.c2 s, A2 = c0.c1 + c1.c2 s, and
//   f^2 = (3 A0^2 - 2 conj A0) + (3 s A2^2 + 2 conj A1) w + (3 A1^2 - 2 conj A2) w^2: 9 Fp2 products instead of 12.
BB_HD void fp4_sqr(const Fp2& a, const Fp2& b, Fp2& r0, Fp2& r1) {   // (a + b s)^2 = (a^2 + xi b^2) + 2ab s
    Fp2 ab = a * b;
    r0 = (a + b) * (a + fp2_mul_xi(b)) - ab - fp2_mul_xi(ab);
    r1 = ab + ab;
}
BB_HD_NOINLINE Fp12 fp12_cyclotomic_sqr(Fp12 f) {
    Fp2 t0, t1, t2, t3, t4, t5;
    fp4_sqr(f.c0.c0, f.c1.c1, t0, t1);     // A0^2
    fp4_sqr(f.c1.c0, f.c0.c2, t2, t3);     // A1^2
    fp4_sqr(f.c0.c1, f.c1.c2, t4, t5);     // A2^2
    auto three_minus_two = [](const Fp2& t, const Fp2& z) { Fp2 d = t - z; return d + d + t; };   // 3t - 2z
    auto three_plus_two = [](const Fp2& t, const Fp2& z) { Fp2 d = t + z; return d + d + t; };    // 3t + 2z
    Fp12 r;
    r.c0.c0 = three_minus_two(t0, f.c0.c0);
    r.c1.c1 = three_plus_two(t1, f.c1.c1);
    r.c1.c0 = three_plus_two(fp2_mul_xi(t5), f.c1.c0);
    r.c0.c2 = three_minus_two(t4, f.c0.c2);
    r.c0.c1 = three_minus_two(t2, f.c0.c1);
    r.c1.c2 = three_plus_two(t3, f.c1.c2);
    return r;
}

// Frobenius f^p: coefficient k of the Fp2[w] view becomes conj(a_k) * xi^(k (p - 1) / 6)
BB_HD Fp2 frob1_coeff(int k) {
    switch (k) {
        case 1: return {Fp{{BBC_FROB1_1_C0_LIST}}, Fp{{BBC_FROB1_1_C1_LIST}}};
        case 2: return {Fp{{BBC_FROB1_2_C0_LIST}}, Fp{{BBC_FROB1_2_C1_LIST}}};
        case 3: return {Fp{{BBC_FROB1_3_C0_LIST}}, Fp{{BBC_FROB1_3_C1_LIST}}};
        case 4: return {Fp{{BBC_FROB1_4_C0_LIST}}, Fp{{BBC_FROB1_4_C1_LIST}}};
        default: return {Fp{{BBC_FROB1_5_C0_LIST}}, Fp{{BBC_FROB1_5_C1_LIST}}};
    }
}
BB_HD_NOINLINE Fp12 fp12_frob1(Fp12 f) {
    Fp12 r;
    r.c0.c0 = fp2_conj(f.c0.c0);
    r.c1.c0 = fp2_conj(f.c1.c0) * frob1_coeff(1);
    r.c0.c1 = fp2_conj(f.c0.c1) * frob1_coeff(2);
    r.c1.c1 = fp2_conj(f.c1.c1) * frob1_coeff(3);
    r.c0.c2 = fp2_conj(f.c0.c2) * frob1_coeff(4);
    r.c1.c2 = fp2_conj(f.c1.c2) * frob1_coeff(5);
    return r;
}
// f^(p^2) as two p-power maps (a direct form with the Fp coefficients xi^(k (p^2 - 1) / 6) computed wrong values
// on sm_90a with nvcc 12.9 while the same source was right on the host; two maps cost 10 Fp2 products more, twice per
// final exponentiation)
BB_HD Fp12 fp12_frob2(const Fp12& f) { return fp12_frob1(fp12_frob1(f)); }

// g^x for g in the cyclotomic subgroup, x = -|x|: 63 cyclotomic squarings, 5 products, one conjugation
BB_HD Fp12 fp12_cyclotomic_exp_x(const Fp12& g) {
    Fp12 r = g;
    for (int i = 62; i >= 0; i--) {
        r = fp12_cyclotomic_sqr(r);
        if ((bbc::BLS_X_ABS >> i) & 1) r = fp12_mul(r, g);
    }
    return r.conj();
}

// f^(3 (p^12 - 1) / r).  Easy part f^((p^6 - 1)(p^2 + 1)), then the x-chain of the hard part.  f != 0.
BB_HD Fp12 fp12_final_exp(const Fp12& f) {
    Fp12 t = fp12_mul(f.conj(), fp12_inv(f));
    t = fp12_mul(fp12_frob2(t), t);
    Fp12 a = fp12_mul(fp12_cyclotomic_exp_x(t), t.conj());             // t^(x - 1)
    a = fp12_mul(fp12_cyclotomic_exp_x(a), a.conj());                  // t^((x - 1)^2)
    Fp12 b = fp12_mul(fp12_cyclotomic_exp_x(a), fp12_frob1(a));        // a^(x + p)
    Fp12 c = fp12_mul(fp12_cyclotomic_exp_x(fp12_cyclotomic_exp_x(b)), fp12_mul(fp12_frob2(b), b.conj()));   // b^(x^2 + p^2 - 1)
    return fp12_mul(c, fp12_mul(fp12_cyclotomic_sqr(t), t));          // * t^3
}

// ---- Miller loop ----------------------------------------------------------------------------------------
// The G1 argument as the lines need it: P = (x / s', y / s'') is passed as x = X ZZZ, y = Y ZZ, s = ZZ ZZZ of
// its XYZZ form (affine: x, y, 1), i.e. every line is evaluated at P times the Fp factor ZZ ZZZ, which the
// final exponentiation removes.  s = 0 marks the identity.
struct G1Eval {
    Fp x, y, s;
};
BB_HD G1Eval g1_eval_from_xyzz(const G1X& p) {
    if (p.is_identity()) return {Fp::zero(), Fp::zero(), Fp::zero()};
    return {p.X * p.ZZZ, p.Y * p.ZZ, p.ZZ * p.ZZZ};
}
BB_HD G1Eval g1_eval_from_affine(const G1Affine& p) {
    if (p.is_identity()) return {Fp::zero(), Fp::zero(), Fp::zero()};
    return {p.x, p.y, fp_one()};
}

// b' = 4 (u + 1), the twist's constant, times k
BB_HD Fp2 twist_b_times(const Fp2& z2, int k) {       // k * b' * z2
    Fp2 t = fp2_mul_xi(z2);
    t = t.dbl().dbl();
    Fp2 r = Fp2::zero();
    for (int i = 0; i < k; i++) r = r + t;
    return r;
}

// T = (X : Y : Z) homogeneous on E': y^2 = x^3 + b'.  Tangent at T evaluated at P, times 2 Y Z^2 w^3 (factors the
// final exponentiation removes): l = (Y^2 - 3 b' Z^2) - 3 X^2 x_P w^2 + 2 Y Z y_P w^3 = (A + B v) + (C v) w.
// T <- 2T as (2XY (Y^2 - 9 b' Z^2) : (Y^2 + 9 b' Z^2)^2 - 108 b'^2 Z^4 : 8 Y^3 Z).
struct G2Proj {
    Fp2 X, Y, Z;
};
// The steps take and return everything by value: nvcc 12.9 has dropped stores to a kernel-local object whose address
// was handed to a non-inlined function (curve.cuh), so no out-of-line function here writes through a reference.
struct MillerStep {
    G2Proj T;
    Fp2 A, B, C;
};
BB_HD_NOINLINE MillerStep miller_dbl_step(G2Proj T, G1Eval p) {
    Fp2 A, B, C;
    Fp2 YY = T.Y.sqr(), ZZ = T.Z.sqr(), XX = T.X.sqr();
    Fp2 b3 = twist_b_times(ZZ, 3);                       // 3 b' Z^2
    A = fp2_mul_fp(YY - b3, p.s);
    B = fp2_mul_fp((XX.dbl() + XX).neg(), p.x);
    Fp2 YZ = T.Y * T.Z;
    C = fp2_mul_fp(YZ.dbl(), p.y);
    Fp2 b9 = b3.dbl() + b3;
    Fp2 XY = T.X * T.Y;
    Fp2 s = YY + b9;
    Fp2 b3sq = b3.sqr();                                 // 9 b'^2 Z^4; 108 b'^2 Z^4 = 12 of it
    Fp2 b12 = b3sq.dbl().dbl();
    G2Proj R;
    R.X = XY.dbl() * (YY - b9);
    R.Y = s.sqr() - (b12.dbl() + b12);
    R.Z = (YY * YZ).dbl().dbl().dbl();
    return {R, A, B, C};
}
// Line through T and Q (affine) at P, times (X - x_Q Z) w^3: l = (theta x_Q - lambda y_Q) - theta x_P w^2 + lambda y_P w^3
// with theta = Y - y_Q Z, lambda = X - x_Q Z.  T <- T + Q.
BB_HD_NOINLINE MillerStep miller_add_step(G2Proj T, G2Affine q, G1Eval p) {
    Fp2 A, B, C;
    Fp2 th = T.Y - q.y * T.Z, la = T.X - q.x * T.Z;
    A = fp2_mul_fp(th * q.x - la * q.y, p.s);
    B = fp2_mul_fp(th.neg(), p.x);
    C = fp2_mul_fp(la, p.y);
    Fp2 la2 = la.sqr(), la3 = la2 * la, la2X = la2 * T.X;
    Fp2 D = th.sqr() * T.Z - la2X.dbl() + la3;
    G2Proj R;
    R.X = la * D;
    R.Y = th * (la2X - D) - T.Y * la3;
    R.Z = la3 * T.Z;
    return {R, A, B, C};
}

// f_{|x|,Q}(P): 63 doubling steps and 5 addition steps.  An identity on either side gives 1 (multi_miller_loop
// skips such pairs).
BB_HD Fp12 miller_loop(const G1Eval& p, const G2Affine& q) {
    if (p.s.is_zero() || q.is_identity()) return Fp12::one();
    G2Proj T{q.x, q.y, fp2_one()};
    Fp12 f = Fp12::one();
    for (int i = 62; i >= 0; i--) {
        f = fp12_sqr(f);
        MillerStep d = miller_dbl_step(T, p);
        T = d.T;
        f = fp12_mul_line(f, d.A, d.B, d.C);
        if ((bbc::BLS_X_ABS >> i) & 1) {
            MillerStep a = miller_add_step(T, q, p);
            T = a.T;
            f = fp12_mul_line(f, a.A, a.B, a.C);
        }
    }
    return f;
}

}  // namespace bb
