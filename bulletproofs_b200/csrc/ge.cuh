// Ristretto255 group operations for the MSM kernels (extended twisted-Edwards coordinates, a = -1).
//
// Replaces, for the device path, what the reference obtains from curve25519_dalek::ristretto /
// ::edwards through the trait calls listed in SURVEY.md §8(b):
//   CompressedRistretto::decompress  -> ge_decode          (src/range_proof/mod.rs:433-443)
//   RistrettoPoint::compress         -> ge_encode          (src/inner_product_proof.rs:99,113)
//   IsIdentity::is_identity          -> ge_is_identity     (src/range_proof/mod.rs:447)
//   RistrettoPoint::from_uniform_bytes -> ge_from_uniform  (src/generators.rs:94-99)
// Formulas are the published ristretto255 / HWCD'08 ones (SURVEY.md §8c recipe), written for one
// thread = one point operation: a warp carries 32 independent bucket or point operations.
#pragma once
#include "fe.cuh"

#define FE_D_LIMBS {0x135978a3u, 0x75eb4dcau, 0x4141d8abu, 0x00700a4du, 0x7779e898u, 0x8cc74079u, 0x2b6ffe73u, 0x52036ceeu}
#define FE_D2_LIMBS {0x26b2f159u, 0xebd69b94u, 0x8283b156u, 0x00e0149au, 0xeef3d130u, 0x198e80f2u, 0x56dffce7u, 0x2406d9dcu}
#define FE_SQRT_M1_LIMBS {0x4a0ea0b0u, 0xc4ee1b27u, 0xad2fe478u, 0x2f431806u, 0x3dfbd7a7u, 0x2b4d0099u, 0x4fc1df0bu, 0x2b832480u}
#define FE_SQRT_AD_MINUS_ONE_LIMBS {0x497b2e1bu, 0x7e97f6a0u, 0x1b7854bdu, 0xaf9d8e0cu, 0x31f5d1fdu, 0x0f3cfcc9u, 0x2b8348acu, 0x376931bfu}
#define FE_INVSQRT_A_MINUS_D_LIMBS {0x805d40eau, 0x99c8fdaau, 0x5a4172beu, 0x9d2f1617u, 0xfe01d840u, 0x16c27b91u, 0xcfaffca2u, 0x786c8905u}
#define FE_ONE_MINUS_D_SQ_LIMBS {0x945fc176u, 0xe27c09c1u, 0xcd5e350fu, 0x2c81a138u, 0xbe70dfe4u, 0x9994abddu, 0xb2b3e0d7u, 0x029072a8u}
#define FE_D_MINUS_ONE_SQ_LIMBS {0x44ed4d20u, 0x31ad5aaau, 0xb01e1999u, 0xd29e4a2cu, 0x529b4eebu, 0x4cdcd32fu, 0xf66c2241u, 0x5968b37au}

BP_HD fe fe_const_d() { return fe{FE_D_LIMBS}; }
BP_HD fe fe_const_d2() { return fe{FE_D2_LIMBS}; }
BP_HD fe fe_const_sqrt_m1() { return fe{FE_SQRT_M1_LIMBS}; }

struct ge_ext { fe X, Y, Z, T; };          // extended (X:Y:Z:T), x = X/Z, y = Y/Z, T = XY/Z
struct ge_niels { fe ypx, ymx, xy2d; };    // affine Niels form of a Z = 1 point: (y+x, y-x, 2d*x*y)

BP_HD ge_ext ge_identity() { ge_ext r; r.X = fe_zero(); r.Y = fe_one(); r.Z = fe_one(); r.T = fe_zero(); return r; }
BP_HD ge_niels ge_niels_identity() { ge_niels r; r.ypx = fe_one(); r.ymx = fe_one(); r.xy2d = fe_zero(); return r; }

// p + q with q affine-Niels: 7 multiplications
BP_HD ge_ext ge_madd(const ge_ext &p, const ge_niels &q) {
    fe A = fe_mul(fe_sub(p.Y, p.X), q.ymx);
    fe B = fe_mul(fe_add(p.Y, p.X), q.ypx);
    fe C = fe_mul(p.T, q.xy2d);
    fe D = fe_dbl(p.Z);
    fe E = fe_sub(B, A), F = fe_sub(D, C), G = fe_add(D, C), H = fe_add(B, A);
    ge_ext r; r.X = fe_mul(E, F); r.Y = fe_mul(G, H); r.T = fe_mul(E, H); r.Z = fe_mul(F, G);
    return r;
}
// p - q with q affine-Niels
BP_HD ge_ext ge_msub(const ge_ext &p, const ge_niels &q) {
    fe A = fe_mul(fe_sub(p.Y, p.X), q.ypx);
    fe B = fe_mul(fe_add(p.Y, p.X), q.ymx);
    fe C = fe_mul(p.T, q.xy2d);
    fe D = fe_dbl(p.Z);
    fe E = fe_sub(B, A), F = fe_add(D, C), G = fe_sub(D, C), H = fe_add(B, A);
    ge_ext r; r.X = fe_mul(E, F); r.Y = fe_mul(G, H); r.T = fe_mul(E, H); r.Z = fe_mul(F, G);
    return r;
}
// p + q, both extended: 9 multiplications
BP_HD ge_ext ge_add(const ge_ext &p, const ge_ext &q) {
    fe A = fe_mul(fe_sub(p.Y, p.X), fe_sub(q.Y, q.X));
    fe B = fe_mul(fe_add(p.Y, p.X), fe_add(q.Y, q.X));
    fe C = fe_mul(fe_mul(p.T, q.T), fe_const_d2());
    fe D = fe_dbl(fe_mul(p.Z, q.Z));
    fe E = fe_sub(B, A), F = fe_sub(D, C), G = fe_add(D, C), H = fe_add(B, A);
    ge_ext r; r.X = fe_mul(E, F); r.Y = fe_mul(G, H); r.T = fe_mul(E, H); r.Z = fe_mul(F, G);
    return r;
}
BP_HD ge_ext ge_neg(const ge_ext &p) { ge_ext r; r.X = fe_neg(p.X); r.Y = p.Y; r.Z = p.Z; r.T = fe_neg(p.T); return r; }
BP_HD ge_ext ge_sub(const ge_ext &p, const ge_ext &q) { return ge_add(p, ge_neg(q)); }
// 2p: 4 squarings + 4 multiplications
BP_HD ge_ext ge_dbl(const ge_ext &p) {
    fe A = fe_sq(p.X), B = fe_sq(p.Y), C = fe_dbl(fe_sq(p.Z));
    fe H = fe_add(A, B);
    fe E = fe_sub(fe_sq(fe_add(p.X, p.Y)), H);
    fe G = fe_sub(B, A);
    fe F = fe_sub(G, C);
    fe Hn = fe_neg(H);
    ge_ext r; r.X = fe_mul(E, F); r.Y = fe_mul(G, Hn); r.T = fe_mul(E, Hn); r.Z = fe_mul(F, G);
    return r;
}
BP_HD ge_niels ge_to_niels_affine(const fe &x, const fe &y) {
    ge_niels r; r.ypx = fe_add(y, x); r.ymx = fe_sub(y, x); r.xy2d = fe_mul(fe_mul(x, y), fe_const_d2()); return r;
}
BP_HD ge_ext ge_from_niels(const ge_niels &n) {   // back to extended (Z = 1); x = (ypx - ymx)/2, y = (ypx + ymx)/2
    return ge_madd(ge_identity(), n);
}
BP_HD ge_niels ge_niels_neg(const ge_niels &n) { ge_niels r; r.ypx = n.ymx; r.ymx = n.ypx; r.xy2d = fe_neg(n.xy2d); return r; }

// Ristretto identity test: the point lies in the identity coset  <=>  X == 0 or Y == 0
BP_HD bool ge_is_identity(const ge_ext &p) { return fe_is_zero(p.X) || fe_is_zero(p.Y); }
BP_HD bool ge_ristretto_eq(const ge_ext &a, const ge_ext &b) {
    return fe_eq(fe_mul(a.X, b.Y), fe_mul(a.Y, b.X)) || fe_eq(fe_mul(a.Y, b.Y), fe_mul(a.X, b.X));
}

// (was_square, r): r = sqrt(u/v) if u/v is square, else sqrt(i*u/v); r is the non-negative root
BP_HDN bool fe_sqrt_ratio_i(fe &r, const fe &u, const fe &v) {
    fe v3 = fe_mul(fe_sq(v), v);
    fe v7 = fe_mul(fe_sq(v3), v);
    fe rr = fe_mul(fe_mul(u, v3), fe_pow22523(fe_mul(u, v7)));
    fe chk = fe_mul(v, fe_sq(rr));
    fe neg_u = fe_neg(u);
    bool ok = fe_eq(chk, u), flip = fe_eq(chk, neg_u), flip_i = fe_eq(chk, fe_mul(neg_u, fe_const_sqrt_m1()));
    rr = fe_select(rr, fe_mul(rr, fe_const_sqrt_m1()), flip || flip_i);
    r = fe_abs(rr);
    return ok || flip;
}

// decode 32 bytes; returns false for anything the reference's decompress() maps to None
BP_HD bool ge_decode(fe &x, fe &y, const uint8_t s_bytes[32]) {
    fe s = fe_frombytes_raw(s_bytes);
    fe sc = fe_canon(s);
    bool canonical = true;
    for (int i = 0; i < 8; i++) canonical &= (sc.v[i] == s.v[i]);      // rejects s >= p and bit 255
    bool neg = s.v[0] & 1u;
    fe one = fe_one();
    fe ss = fe_sq(s), u1 = fe_sub(one, ss), u2 = fe_add(one, ss), u2s = fe_sq(u2);
    fe v = fe_sub(fe_neg(fe_mul(fe_const_d(), fe_sq(u1))), u2s);
    fe I;
    bool ok = fe_sqrt_ratio_i(I, one, fe_mul(v, u2s));
    fe dx = fe_mul(I, u2), dy = fe_mul(fe_mul(I, dx), v);
    x = fe_abs(fe_mul(fe_dbl(s), dx));
    y = fe_mul(u1, dy);
    fe t = fe_mul(x, y);
    return canonical && !neg && ok && !fe_is_negative(t) && !fe_is_zero(y);
}

BP_HD void ge_encode(uint8_t out[32], const ge_ext &p) {
    fe u1 = fe_mul(fe_add(p.Z, p.Y), fe_sub(p.Z, p.Y));
    fe u2 = fe_mul(p.X, p.Y);
    fe I;
    fe_sqrt_ratio_i(I, fe_one(), fe_mul(u1, fe_sq(u2)));
    fe d1 = fe_mul(I, u1), d2 = fe_mul(I, u2);
    fe zinv = fe_mul(fe_mul(d1, d2), p.T);
    fe ix = fe_mul(p.X, fe_const_sqrt_m1()), iy = fe_mul(p.Y, fe_const_sqrt_m1());
    fe ench = fe_mul(d1, fe{FE_INVSQRT_A_MINUS_D_LIMBS});
    bool rot = fe_is_negative(fe_mul(p.T, zinv));
    fe x = fe_select(p.X, iy, rot), y = fe_select(p.Y, ix, rot), dinv = fe_select(d2, ench, rot);
    y = fe_cneg(y, fe_is_negative(fe_mul(x, zinv)));
    fe s = fe_abs(fe_mul(dinv, fe_sub(p.Z, y)));
    fe_tobytes(out, s);
}

// Elligator map of one field element (ristretto flavour)
BP_HD ge_ext ge_elligator(const fe &r0) {
    fe one = fe_one(), d = fe_const_d();
    fe r = fe_mul(fe_const_sqrt_m1(), fe_sq(r0));
    fe Ns = fe_mul(fe_add(r, one), fe{FE_ONE_MINUS_D_SQ_LIMBS});
    fe c = fe_neg(one);
    fe D = fe_mul(fe_sub(c, fe_mul(d, r)), fe_add(r, d));
    fe s;
    bool sq = fe_sqrt_ratio_i(s, Ns, D);
    fe sp = fe_mul(s, r0);
    sp = fe_cneg(sp, !fe_is_negative(sp));
    s = fe_select(s, sp, !sq);
    c = fe_select(c, r, !sq);
    fe Nt = fe_sub(fe_mul(fe_mul(c, fe_sub(r, one)), fe{FE_D_MINUS_ONE_SQ_LIMBS}), D);
    fe ss = fe_sq(s);
    fe w0 = fe_mul(fe_dbl(s), D), w1 = fe_mul(Nt, fe{FE_SQRT_AD_MINUS_ONE_LIMBS}), w2 = fe_sub(one, ss), w3 = fe_add(one, ss);
    ge_ext p; p.X = fe_mul(w0, w3); p.Y = fe_mul(w2, w1); p.Z = fe_mul(w1, w3); p.T = fe_mul(w0, w2);
    return p;
}
// RistrettoPoint::from_uniform_bytes: two Elligator maps (bit 255 of each half ignored) and one addition
BP_HD ge_ext ge_from_uniform(const uint8_t b[64]) {
    fe r1 = fe_frombytes_raw(b), r2 = fe_frombytes_raw(b + 32);
    r1.v[7] &= 0x7fffffffu; r2.v[7] &= 0x7fffffffu;
    return ge_add(ge_elligator(r1), ge_elligator(r2));
}
