// b2k_rne_gen.cpp -- robot-specialised code generation for the recursive Newton-Euler kernels.
//
// The generic kernels (b2k_rne.cuh) multiply through every link parameter of the 24-double table
// whether it is zero or not: for a Puma560 that is 886 FP64 instructions per row, and the kernel is
// FP64-pipe bound.  Most of a real arm's table is structure, not numbers:
// alpha in {0, +-pi/2}, a or d zero, centre of mass on an axis, diagonal inertia, no tip wrench, gravity
// along one base axis, and the first links of the chain carry sparse velocities (w_0 = 0).  This file
// is the chain compiler for dynamics: it runs the Luh-Walker-Paul recursion (reference ne.c:137-457)
// SYMBOLICALLY over scalars that are either exactly zero, a known constant or a run-time value, and
// emits straight-line CUDA C in which a term whose factor is zero never appears, a factor of +-1 is
// a sign, constants are folded, and every sum of products is a chain of FMAs.  The text is compiled
// for sm_90a at run time (NVRTC, b2k_rne_spec.cu) into a kernel for THIS robot; the same text
// compiles as plain C++ for the host, which is how tests/ check it against the oracle without a GPU.
//
// The dynamics fan-outs of the reference's DynamicsMixin (Dynamics.py: inertia, gravload, itorque,
// coriolis, accel) are the same recursion evaluated with symbolic unit / zero inputs, so e.g. the
// column i of the inertia matrix costs only the links i..n-1 and nothing of the velocity terms.
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <functional>
#include <map>
#include <string>
#include <vector>

#include "b2k_rne_gen.h"

namespace {

// ------------------------------------------------------------------ symbolic scalars
struct Opd { // an operand an instruction can take directly: a run-time variable or a constant-bank entry
    bool isc = false;
    double c = 0.0; // constant value (isc)
    int id = -1;    // variable id (!isc)
    bool neg = false;
};
struct Sym {
    enum Kind { Z, O, P } k = Z; // zero | operand | pending product x*y (sign in x)
    Opd x, y;
};

// How an emitted variable was computed, kept so that its derivatives can be emitted afterwards (tangent()):
// a * b, fma(a, b, c), a + b (signs in the operands), or a leaf -- a named input or a term with no derivative rule.
struct Def {
    enum Op { LEAF, MUL, FMA, ADD } op = LEAF;
    Opd a, b, c;
};

struct Gen {
    std::vector<std::string> code;
    std::vector<std::string> names; // variable id -> spelling
    std::vector<Def> defs;          // variable id -> how it was computed
    std::vector<double> consts;     // constant bank
    std::map<unsigned long long, int> cslot;
    int n_mul = 0, n_fma = 0, n_add = 0;

    int new_var(const Def &d = Def())
    {
        names.push_back("t" + std::to_string((int)names.size()));
        defs.push_back(d);
        return (int)names.size() - 1;
    }
    int named_var(const std::string &s)
    {
        names.push_back(s);
        defs.push_back(Def());
        return (int)names.size() - 1;
    }
    static Sym zero() { return Sym(); }
    static Sym cst(double c)
    {
        Sym s;
        if (c == 0.0) return s;
        s.k = Sym::O; s.x.isc = true; s.x.c = c;
        return s;
    }
    Sym var(const std::string &name)
    {
        Sym s;
        s.k = Sym::O; s.x.id = named_var(name);
        return s;
    }
    std::string spell(const Opd &o, bool flip = false)
    {
        bool neg = o.neg != flip;
        if (o.isc) {
            double v = o.c;
            if (v < 0) { v = -v; neg = !neg; }
            unsigned long long bits;
            memcpy(&bits, &v, 8);
            auto it = cslot.find(bits);
            int slot;
            if (it == cslot.end()) { slot = (int)consts.size(); consts.push_back(v); cslot[bits] = slot; }
            else slot = it->second;
            return std::string(neg ? "-" : "") + "C[" + std::to_string(slot) + "]";
        }
        return std::string(neg ? "-" : "") + names[o.id];
    }
    Sym emit(const std::string &rhs, const Def &d = Def())
    {
        int id = new_var(d);
        code.push_back("    const real " + names[id] + " = " + rhs + ";");
        Sym s;
        s.k = Sym::O; s.x.id = id;
        return s;
    }
    // a value an instruction can read: pending products are multiplied out
    Opd operand(const Sym &a)
    {
        if (a.k == Sym::O) return a.x;
        Def d;
        d.op = Def::MUL; d.a = a.x; d.b = a.y;
        Sym m = emit(spell(a.x) + " * " + spell(a.y), d);
        n_mul++;
        return m.x;
    }
    Sym neg(Sym a)
    {
        if (a.k == Sym::Z) return a;
        if (a.x.isc) a.x.c = -a.x.c;
        else a.x.neg = !a.x.neg;
        return a;
    }
    Sym mul(const Sym &a, const Sym &b)
    {
        if (a.k == Sym::Z || b.k == Sym::Z) return zero();
        Opd x = operand(a), y = operand(b);
        if (x.isc && x.neg) { x.c = -x.c; x.neg = false; }
        if (y.isc && y.neg) { y.c = -y.c; y.neg = false; }
        if (x.isc && y.isc) return cst(x.c * y.c);
        if (y.isc) std::swap(x, y); // constant first
        if (x.isc && (x.c == 1.0 || x.c == -1.0)) {
            Sym s;
            s.k = Sym::O; s.x = y;
            if (x.c < 0) s = neg(s);
            return s;
        }
        Sym s;
        s.k = Sym::P;
        if (x.isc) std::swap(x, y); // keep the variable in x, the constant in y
        s.x = x; s.y = y;
        if (s.y.neg) { s.y.neg = false; s.x.neg = !s.x.neg; }
        if (s.y.isc && s.y.c < 0) { s.y.c = -s.y.c; s.x.neg = !s.x.neg; }
        return s;
    }
    // n-ary sum: constants folded, one chain of FMAs over the products, plain additions last
    Sym sum(const std::vector<Sym> &terms)
    {
        double K = 0.0;
        std::vector<Opd> plain;
        std::vector<Sym> prods;
        for (const Sym &t : terms) {
            if (t.k == Sym::Z) continue;
            if (t.k == Sym::P) { prods.push_back(t); continue; }
            if (t.x.isc) K += t.x.c;
            else plain.push_back(t.x);
        }
        if (K != 0.0) { Opd o; o.isc = true; o.c = K; plain.push_back(o); }
        if (plain.empty() && prods.empty()) return zero();
        if (plain.size() + prods.size() == 1) {
            if (!prods.empty()) return prods[0];
            Sym s; s.k = Sym::O; s.x = plain[0];
            return s;
        }
        Opd acc;
        size_t pi = 0, ai = 0;
        if (!plain.empty()) { acc = plain[0]; ai = 1; }
        else { acc = operand(prods[0]); pi = 1; }
        for (; pi < prods.size(); pi++) {
            Def d;
            d.op = Def::FMA; d.a = prods[pi].x; d.b = prods[pi].y; d.c = acc;
            acc = emit("fma(" + spell(prods[pi].x) + ", " + spell(prods[pi].y) + ", " + spell(acc) + ")", d).x;
            n_fma++;
        }
        for (; ai < plain.size(); ai++) {
            const Opd &b = plain[ai];
            const bool bneg = b.isc ? ((b.c < 0) != b.neg) : b.neg;
            Opd babs = b;
            babs.neg = false;
            if (babs.isc) babs.c = fabs(babs.c);
            std::string rhs;
            rhs = spell(acc) + (bneg ? " - " : " + ") + spell(babs);
            Def d;
            d.op = Def::ADD; d.a = acc; d.b = b;
            acc = emit(rhs, d).x;
            n_add++;
        }
        Sym s; s.k = Sym::O; s.x = acc;
        return s;
    }
    Sym add(const Sym &a, const Sym &b) { return sum({a, b}); }
    Sym sub(const Sym &a, const Sym &b) { return sum({a, neg(b)}); }
    // make sure a value that will be read several times is not a pending product
    Sym fix(const Sym &a)
    {
        if (a.k != Sym::P) return a;
        Sym s; s.k = Sym::O; s.x = operand(a);
        return s;
    }
    static Sym val(const Opd &o)
    {
        if (o.isc) return cst(o.neg ? -o.c : o.c);
        Sym s; s.k = Sym::O; s.x = o;
        return s;
    }
    // Forward-mode derivative of the variables emitted so far along one direction.  seed[id] is the derivative of the
    // leaf variable id (zero when unset); returns the derivative of every variable below `upto`.  The product rule
    // runs through mul / sum, so a factor whose derivative is structurally zero drops out: no instruction is emitted
    // for a variable that does not depend on the direction.
    std::vector<Sym> tangent(int upto, const std::vector<Sym> &seed)
    {
        std::vector<Sym> T(seed);
        T.resize(upto);
        auto dt = [&](const Opd &o) { // the derivative of an operand (a pending product is read as a plain variable)
            if (o.isc) return zero();
            return o.neg ? neg(T[o.id]) : T[o.id];
        };
        auto dtf = [&](const Opd &o) { // ... when it becomes a factor: multiplied out once, then reused
            if (o.isc) return zero();
            T[o.id] = fix(T[o.id]);
            return o.neg ? neg(T[o.id]) : T[o.id];
        };
        for (int id = 0; id < upto; id++) {
            const Def d = defs[id]; // a copy: the rules below emit, and emit() grows defs
            switch (d.op) {
            case Def::LEAF: break;
            case Def::MUL: T[id] = sum({mul(dtf(d.a), val(d.b)), mul(val(d.a), dtf(d.b))}); break;
            case Def::FMA: T[id] = sum({mul(dtf(d.a), val(d.b)), mul(val(d.a), dtf(d.b)), dt(d.c)}); break;
            case Def::ADD: T[id] = sum({dt(d.a), dt(d.b)}); break;
            }
        }
        return T;
    }
};

struct V3 { Sym x, y, z; };

struct Vops {
    Gen &g;
    explicit Vops(Gen &gg) : g(gg) {}
    V3 zero() { return {Gen::zero(), Gen::zero(), Gen::zero()}; }
    V3 cst(const double *v) { return {Gen::cst(v[0]), Gen::cst(v[1]), Gen::cst(v[2])}; }
    V3 fix(const V3 &a) { return {g.fix(a.x), g.fix(a.y), g.fix(a.z)}; }
    V3 add(const V3 &a, const V3 &b) { return {g.add(a.x, b.x), g.add(a.y, b.y), g.add(a.z, b.z)}; }
    V3 scale(const Sym &s, const V3 &a) { return {g.mul(s, a.x), g.mul(s, a.y), g.mul(s, a.z)}; }
    // a x b + c (+ d), each component one FMA chain
    V3 cross_acc(const V3 &a, const V3 &b, const V3 *c = nullptr, const V3 *d = nullptr)
    {
        V3 A = fix(a), B = fix(b);
        auto comp = [&](const Sym &p, const Sym &q, const Sym &r, const Sym &s, const Sym *e, const Sym *f) {
            std::vector<Sym> t = {g.mul(p, q), g.neg(g.mul(r, s))};
            if (e) t.push_back(*e);
            if (f) t.push_back(*f);
            return g.sum(t);
        };
        return {comp(A.y, B.z, A.z, B.y, c ? &c->x : nullptr, d ? &d->x : nullptr),
                comp(A.z, B.x, A.x, B.z, c ? &c->y : nullptr, d ? &d->y : nullptr),
                comp(A.x, B.y, A.y, B.x, c ? &c->z : nullptr, d ? &d->z : nullptr)};
    }
    // planar rotations: Rz(th) v and Rz(-th) v with run-time (s, c); Rx(al) v and Rx(-al) v with (sa, ca)
    V3 rotz(const Sym &s, const Sym &c, const V3 &v, bool transpose, const V3 *acc = nullptr)
    {
        V3 a = fix(v);
        const Sym sx = transpose ? s : g.neg(s);
        // [c -s; s c] (or its transpose [c s; -s c]) on (x, y)
        return {g.sum({g.mul(c, a.x), g.mul(sx, a.y), acc ? acc->x : Gen::zero()}),
                g.sum({g.mul(g.neg(sx), a.x), g.mul(c, a.y), acc ? acc->y : Gen::zero()}),
                acc ? g.add(a.z, acc->z) : a.z};
    }
    V3 rotx(const Sym &s, const Sym &c, const V3 &v, bool transpose, const V3 *acc = nullptr)
    {
        V3 a = fix(v);
        const Sym sx = transpose ? s : g.neg(s);
        return {acc ? g.add(a.x, acc->x) : a.x,
                g.sum({g.mul(c, a.y), g.mul(sx, a.z), acc ? acc->y : Gen::zero()}),
                g.sum({g.mul(g.neg(sx), a.y), g.mul(c, a.z), acc ? acc->z : Gen::zero()})};
    }
    V3 matvec(const double *I /* row-major 3x3, read column-major like vmath.c mat_vect_mult */, const V3 &v)
    {
        V3 a = fix(v);
        auto row = [&](int r) {
            return g.sum({g.mul(Gen::cst(I[r]), a.x), g.mul(Gen::cst(I[3 + r]), a.y), g.mul(Gen::cst(I[6 + r]), a.z)});
        };
        return {row(0), row(1), row(2)};
    }
};

double snap(double v)
{ // sin / cos of alpha = k pi/2 come out of libm as 6.1e-17 or 1 - 1e-16: structure, not numbers
    const double r = nearbyint(v);
    if (fabs(v - r) < 4e-16 && fabs(r) <= 1.0) return r;
    return v;
}

struct Link {
    Sym st, ct, sa, ca; // joint rotation (run time; constants of theta for a prismatic link), twist (constants)
    bool pris = false;
    V3 ps;              // p*: (a, d sin(alpha), d cos(alpha)) for DH, (a, -d sin(alpha), d cos(alpha)) for MDH; d = q + offset if prismatic
    double r[3], I[9], m, c_jm, c_b, c_tcp, c_tcm;
};

struct Inputs { // one evaluation of the recursion: per-joint velocity / acceleration symbols, base acceleration, tip wrench
    std::vector<Sym> qd, qdd;
    V3 grav, ftip, ntip;
    bool friction = true;
    bool wrench = false; // also return the base wrench (6 symbols after the n torques)
};

// One Luh-Walker-Paul recursion over symbolic inputs; returns the joint torques as symbols.
// Standard DH: reference ne.c:245-347 (forward), 409-457 (backward); modified DH: ne.c:137-240, 358-403;
// joint torque with the actuator terms: ne.c:464-491.  All-revolute chains.
std::vector<Sym> recursion(Gen &g, const std::vector<Link> &L, bool mdh, const Inputs &in)
{
    Vops v(g);
    const int N = (int)L.size();
    std::vector<V3> Fm(N), Nm(N);
    V3 w = v.zero(), wd = v.zero(), acc = v.zero();
    auto RT = [&](const Link &l, const V3 &a, const V3 *add = nullptr) { // R^T a (+ add)
        if (!mdh) return v.rotx(l.sa, l.ca, v.rotz(l.st, l.ct, a, true), true, add); // R = Rz(th) Rx(al)
        return v.rotz(l.st, l.ct, v.rotx(l.sa, l.ca, a, true), true, add);          // R = Rx(al) Rz(th)
    };
    auto R = [&](const Link &l, const V3 &a, const V3 *add = nullptr) { // R a (+ add)
        if (!mdh) return v.rotz(l.st, l.ct, v.rotx(l.sa, l.ca, a, false), false, add);
        return v.rotx(l.sa, l.ca, v.rotz(l.st, l.ct, a, false), false, add);
    };
    for (int j = 0; j < N; j++) {
        const Link &l = L[j];
        const V3 ps = l.ps, rc = v.cst(l.r);
        const Sym qd = in.qd[j], qdd = in.qdd[j];
        V3 wn, wdn, accn;
        if (l.pris) { // translational joint along z_{j-1} (ne.c:183-225 MDH, 290-333 DH): no joint rate in w / wd
            const V3 qdv = {Gen::zero(), Gen::zero(), qd}, qddv = {Gen::zero(), Gen::zero(), qdd};
            const Sym two = Gen::cst(2.0);
            if (mdh) {
                if (j == 0) { // sic, ne.c:187-204: the base acceleration is taken over unrotated
                    wn = qdv; wdn = qddv; accn = in.grav;
                } else {
                    wn = RT(l, w);
                    wdn = RT(l, wd);
                    const V3 wxp = v.cross_acc(w, ps);
                    const V3 a = v.cross_acc(wd, ps, &acc);
                    const V3 t = RT(l, v.cross_acc(w, wxp, &a));
                    const V3 c2 = v.scale(two, v.cross_acc(v.fix(wn), qdv));
                    accn = v.add(v.add(t, c2), qddv);
                }
            } else {
                V3 base;
                if (j == 0) { wn = v.zero(); wdn = v.zero(); base = RT(l, v.add(qddv, in.grav)); }
                else { wn = v.fix(RT(l, w)); wdn = v.fix(RT(l, wd)); base = RT(l, v.add(qddv, acc)); }
                const V3 a1 = v.cross_acc(wdn, ps, &base);
                const V3 c2 = v.scale(two, v.cross_acc(wn, RT(l, qdv)));
                const V3 a2 = v.add(a1, c2);
                const V3 wxp = v.cross_acc(wn, ps);
                accn = v.cross_acc(wn, wxp, &a2);
            }
        } else if (mdh) {
            if (j == 0) {
                wn = {Gen::zero(), Gen::zero(), qd};
                wdn = {Gen::zero(), Gen::zero(), qdd};
                accn = RT(l, in.grav);
            } else {
                const V3 t1 = v.fix(RT(l, w));
                wn = {t1.x, t1.y, g.add(t1.z, qd)};
                const V3 t3 = RT(l, wd);
                // t1 x (0,0,qd) + t3 + (0,0,qdd)
                wdn = {g.sum({g.mul(t1.y, qd), t3.x}), g.sum({g.neg(g.mul(t1.x, qd)), t3.y}), g.add(t3.z, qdd)};
                const V3 wxp = v.cross_acc(w, ps);
                const V3 a = v.cross_acc(wd, ps, &acc);
                accn = RT(l, v.cross_acc(w, wxp, &a));
            }
        } else {
            const V3 wz = {w.x, w.y, g.add(w.z, qd)};
            wn = RT(l, wz);
            // wd + (0,0,qdd) + w x (0,0,qd)
            const V3 wdz = {g.sum({g.mul(w.y, qd), wd.x}), g.sum({g.neg(g.mul(w.x, qd)), wd.y}), g.add(wd.z, qdd)};
            wdn = RT(l, wdz);
            wn = v.fix(wn);
            wdn = v.fix(wdn);
            const V3 rg = RT(l, j == 0 ? in.grav : acc);
            const V3 t2 = v.cross_acc(wn, ps);
            const V3 a = v.cross_acc(wdn, ps, &rg);
            accn = v.cross_acc(wn, t2, &a);
        }
        w = v.fix(wn); wd = v.fix(wdn); acc = v.fix(accn);
        const V3 wxr = v.cross_acc(w, rc);
        const V3 a1 = v.cross_acc(wd, rc, &acc);
        const V3 abar = v.cross_acc(w, wxr, &a1);
        Fm[j] = v.fix(v.scale(Gen::cst(l.m), abar));
        const V3 Iw = v.matvec(l.I, w), Iwd = v.matvec(l.I, wd);
        Nm[j] = v.fix(v.cross_acc(w, Iw, &Iwd));
    }
    std::vector<Sym> tau(N);
    V3 f = v.zero(), nn = v.zero();
    for (int j = N - 1; j >= 0; j--) {
        const Link &l = L[j];
        const V3 rc = v.cst(l.r);
        V3 fj, nj;
        const V3 rxF = v.cross_acc(rc, Fm[j], &Nm[j]); // r x F + N
        if (mdh) {
            if (j == N - 1) {
                fj = v.add(in.ftip, Fm[j]);
                nj = v.add(in.ntip, rxF);
            } else {
                const Link &ln = L[j + 1];
                const V3 psn = ln.ps;
                const V3 Rf = v.fix(R(ln, f));
                fj = v.add(Rf, Fm[j]);
                const V3 pxf = v.cross_acc(psn, Rf, &rxF);
                nj = R(ln, nn, &pxf);
            }
        } else {
            const V3 ps = l.ps;
            if (j == N - 1) {
                fj = v.fix(v.add(in.ftip, Fm[j]));
                nj = v.cross_acc(ps, fj, &rxF, &in.ntip);
            } else {
                const Link &ln = L[j + 1];
                fj = v.fix(R(ln, f, &Fm[j]));
                const V3 pxf = v.cross_acc(ps, fj, &rxF);
                nj = R(ln, nn, &pxf);
            }
        }
        f = v.fix(fj); nn = v.fix(nj);
        // torque about (force along, for a prismatic joint) the joint axis z_{j-1} seen from frame j:
        // (0, sa, ca) for DH, (0, 0, 1) for MDH
        std::vector<Sym> t;
        const V3 &load = l.pris ? f : nn;
        if (mdh) t.push_back(load.z);
        else { t.push_back(g.mul(load.y, l.sa)); t.push_back(g.mul(load.z, l.ca)); }
        t.push_back(g.mul(Gen::cst(l.c_jm), in.qdd[j]));
        if (in.friction) t.push_back(g.mul(Gen::cst(l.c_b), in.qd[j]));
        Sym tq = g.fix(g.sum(t));
        if (in.friction && (l.c_tcp != 0.0 || l.c_tcm != 0.0) && in.qd[j].k != Sym::Z) {
            // Coulomb friction, asymmetric, none at rest (ne.c:487-490)
            const Opd qdo = g.operand(in.qd[j]);
            if (qdo.isc) {
                const double c = qdo.c > 0 ? l.c_tcp : (qdo.c < 0 ? l.c_tcm : 0.0);
                tq = g.fix(g.add(tq, Gen::cst(c)));
            } else { // tq + Tc+ [qd > 0] + Tc- [qd < 0]: two FMAs against 0 / 1 masks, no branch
                const std::string q = g.spell(qdo);
                // the Coulomb term is piecewise constant: tangent() reads the result as tq + 0 (tq itself may be a
                // structural zero: a link with no mass, inertia or other actuator term on its axis)
                Def d;
                d.op = Def::ADD; d.b.isc = true;
                if (tq.k == Sym::Z) d.a.isc = true;
                else d.a = g.operand(tq);
                std::string e = tq.k == Sym::Z ? "(real)0" : g.spell(d.a);
                if (l.c_tcm != 0.0) { Opd m; m.isc = true; m.c = l.c_tcm; e = "fma(" + g.spell(m) + ", step_neg(" + q + "), " + e + ")"; g.n_fma++; }
                if (l.c_tcp != 0.0) { Opd p; p.isc = true; p.c = l.c_tcp; e = "fma(" + g.spell(p) + ", step_pos(" + q + "), " + e + ")"; g.n_fma++; }
                tq = g.emit(e, d);
            }
        }
        tau[j] = tq;
    }
    if (in.wrench) { // what the base exerts on link 1, in frame 0: R_1 f_1, R_1 n_1 (+ p*_1 x R_1 f_1 for MDH); b2k_rne.cuh
        const V3 f0 = v.fix(R(L[0], f));
        V3 n0;
        if (mdh) {
            const V3 pxf = v.cross_acc(L[0].ps, f0);
            n0 = R(L[0], nn, &pxf);
        } else {
            n0 = R(L[0], nn);
        }
        for (const Sym &s : {f0.x, f0.y, f0.z, n0.x, n0.y, n0.z}) tau.push_back(s);
    }
    return tau;
}

std::string assign(Gen &g, const std::string &lhs, const Sym &s)
{
    if (s.k == Sym::Z) return "    " + lhs + " = (real)0;";
    return "    " + lhs + " = " + g.spell(g.operand(s)) + ";";
}

// The operations of DynamicsMixin as evaluations of ONE recursion over symbolic inputs (`rec`: per-joint velocity and
// acceleration symbols in q order, base acceleration, tip wrench -> joint torques): shared by the DH recursion and the
// spatial-vector recursion of rigid-body trees.  Fills the statements that store the result (`tail`) and the signature.
typedef std::function<std::vector<Sym>(const Inputs &)> RecFn;
int assemble(Gen &g, int N, const b2k_gen_opts &o, const RecFn &rec, std::vector<std::string> &tail, const char *&sig, std::string &err)
{
    auto jvec = [&](const char *name) {
        std::vector<Sym> s(N);
        for (int j = 0; j < N; j++) s[j] = g.var(std::string(name) + "[" + std::to_string(j) + "]");
        return s;
    };
    auto gvec = [&]() {
        V3 v;
        v.x = (o.grav_mask & 1) ? g.var("grav[0]") : Gen::zero();
        v.y = (o.grav_mask & 2) ? g.var("grav[1]") : Gen::zero();
        v.z = (o.grav_mask & 4) ? g.var("grav[2]") : Gen::zero();
        return v;
    };
    const std::vector<Sym> zeros(N, Gen::zero());
    Vops vo(g);
    Inputs in;
    in.grav = vo.zero(); in.ftip = vo.zero(); in.ntip = vo.zero();
    if (o.mode == B2K_GEN_RNE || o.mode == B2K_GEN_RNE_WRENCH) { // RNE_WRENCH: out = [tau (n) | base wrench (6)]
        sig = "rne_row(const real *C, const real *grav, const real *fext, const real *st, const real *ct, const real *qq, "
              "const real *qd, const real *qdd, real *out)";
        in.qd = jvec("qd"); in.qdd = jvec("qdd");
        in.grav = gvec();
        if (o.has_fext) {
            in.ftip = {g.var("fext[0]"), g.var("fext[1]"), g.var("fext[2]")};
            in.ntip = {g.var("fext[3]"), g.var("fext[4]"), g.var("fext[5]")};
        }
        in.wrench = o.mode == B2K_GEN_RNE_WRENCH;
        std::vector<Sym> tau = rec(in);
        for (int j = 0; j < (int)tau.size(); j++) tail.push_back(assign(g, "out[" + std::to_string(j) + "]", tau[j]));
    } else if (o.mode == B2K_GEN_GRAVLOAD) { // rne(q, 0, 0, g)  Dynamics.py:912-915
        sig = "rne_row(const real *C, const real *grav, const real *fext, const real *st, const real *ct, const real *qq, "
              "const real *in1, const real *in2, real *out)";
        in.qd = zeros; in.qdd = zeros; in.grav = gvec();
        std::vector<Sym> tau = rec(in);
        for (int j = 0; j < N; j++) tail.push_back(assign(g, "out[" + std::to_string(j) + "]", tau[j]));
    } else if (o.mode == B2K_GEN_ITORQUE) { // rne(q, 0, qdd, g = 0)  Dynamics.py:1456-1459
        sig = "rne_row(const real *C, const real *grav, const real *fext, const real *st, const real *ct, const real *qq, "
              "const real *in1, const real *in2, real *out)";
        in.qd = zeros; in.qdd = jvec("in1");
        std::vector<Sym> tau = rec(in);
        for (int j = 0; j < N; j++) tail.push_back(assign(g, "out[" + std::to_string(j) + "]", tau[j]));
    } else if (o.mode == B2K_GEN_INERTIA) { // row i of M = rne(q, 0, e_i, g = 0)  Dynamics.py:752-758
        sig = "rne_row(const real *C, const real *grav, const real *fext, const real *st, const real *ct, const real *qq, "
              "const real *in1, const real *in2, real *out)";
        for (int i = 0; i < N; i++) {
            in.qd = zeros; in.qdd = zeros;
            in.qdd[i] = Gen::cst(1.0);
            std::vector<Sym> tau = rec(in);
            for (int k = 0; k < N; k++) tail.push_back(assign(g, "out[" + std::to_string(i * N + k) + "]", tau[k]));
        }
    } else if (o.mode == B2K_GEN_CORIOLIS) { // Dynamics.py:825-857 on the friction-free robot
        sig = "rne_row(const real *C, const real *grav, const real *fext, const real *st, const real *ct, const real *qq, "
              "const real *in1, const real *in2, real *out)";
        in.friction = false;
        std::vector<Sym> qd = jvec("in1");
        std::vector<std::vector<Sym>> Csq(N, std::vector<Sym>(N));
        std::vector<std::vector<std::vector<Sym>>> terms(N, std::vector<std::vector<Sym>>(N));
        for (int i = 0; i < N; i++) { // centripetal: joint i alone at unit speed
            in.qd = zeros; in.qdd = zeros;
            in.qd[i] = Gen::cst(1.0);
            std::vector<Sym> tau = rec(in);
            for (int k = 0; k < N; k++) Csq[k][i] = g.fix(tau[k]);
        }
        const Sym half = Gen::cst(0.5);
        for (int i = 0; i < N; i++)
            for (int j = i + 1; j < N; j++) { // Coriolis: joints i and j at unit speed
                in.qd = zeros; in.qdd = zeros;
                in.qd[i] = Gen::cst(1.0); in.qd[j] = Gen::cst(1.0);
                std::vector<Sym> tau = rec(in);
                for (int k = 0; k < N; k++) {
                    const Sym t = g.fix(g.sum({tau[k], g.neg(Csq[k][j]), g.neg(Csq[k][i])}));
                    const Sym th = g.fix(g.mul(half, t));
                    terms[k][j].push_back(g.mul(th, qd[i]));
                    terms[k][i].push_back(g.mul(th, qd[j]));
                }
            }
        for (int k = 0; k < N; k++)
            for (int i = 0; i < N; i++) {
                terms[k][i].push_back(g.mul(Csq[k][i], qd[i]));
                tail.push_back(assign(g, "out[" + std::to_string(k * N + i) + "]", g.sum(terms[k][i])));
            }
    } else if (o.mode == B2K_GEN_ACCEL) {
        // tau0 = rne(q, qd, 0, g) with friction; M rows with unit accelerations, no gravity: out = [M (n*n) | torque - tau0 (n)]
        // (the kernel wrapper solves the n x n system; Dynamics.py:490-503)
        sig = "rne_row(const real *C, const real *grav, const real *fext, const real *st, const real *ct, const real *qq, "
              "const real *in1, const real *in2, real *out)";
        in.qd = jvec("in1"); in.qdd = zeros; in.grav = gvec();
        std::vector<Sym> tau0 = rec(in);
        std::vector<Sym> tq = jvec("in2");
        for (int k = 0; k < N; k++) tail.push_back(assign(g, "out[" + std::to_string(N * N + k) + "]", g.sub(tq[k], tau0[k])));
        in.grav = vo.zero();
        for (int i = 0; i < N; i++) {
            in.qd = zeros; in.qdd = zeros;
            in.qdd[i] = Gen::cst(1.0);
            std::vector<Sym> tau = rec(in);
            for (int k = 0; k < N; k++) tail.push_back(assign(g, "out[" + std::to_string(i * N + k) + "]", tau[k]));
        }
    } else if (o.mode == B2K_GEN_RNE_DERIV) {
        // tau = rne(q, qd, qdd, g) once, then one tangent pass per direction q_0..q_{n-1}, qd_0..qd_{n-1}:
        // dq[i * n + k] = d tau_i / d q_k, dqd[i * n + k] = d tau_i / d qd_k.  Each column is stored as soon as its pass
        // ends, so that only one direction's tangents are live at a time.
        sig = "rne_deriv_row(const real *C, const real *grav, const real *fext, const real *st, const real *ct, const real *qq, "
              "const real *qd, const real *qdd, real *dq, real *dqd)";
        in.qd = jvec("qd"); in.qdd = jvec("qdd");
        in.grav = gvec();
        std::vector<Sym> tau = rec(in);
        for (Sym &s : tau) s = g.fix(s);
        const int upto = (int)g.names.size();
        std::map<std::string, int> leaf; // the inputs of this function (the latest leaf of each name)
        for (int id = 0; id < upto; id++)
            if (g.defs[id].op == Def::LEAF && g.names[id].find('[') != std::string::npos) leaf[g.names[id]] = id;
        auto id_of = [&](const char *a, int k) {
            auto it = leaf.find(std::string(a) + "[" + std::to_string(k) + "]");
            return it == leaf.end() ? -1 : it->second;
        };
        auto leafsym = [&](int id) { Opd x; x.id = id; return Gen::val(x); };
        for (int dir = 0; dir < 2 * N; dir++) {
            const int k = dir % N;
            std::vector<Sym> seed(upto);
            if (dir < N) { // st = sin q -> cos q, ct = cos q -> -sin q, qq = q -> 1 (a flipped joint's sign is in the recursion)
                const int is = id_of("st", k), ic = id_of("ct", k), iq = id_of("qq", k);
                if (is >= 0 && ic >= 0) { seed[is] = leafsym(ic); seed[ic] = g.neg(leafsym(is)); }
                if (iq >= 0) seed[iq] = Gen::cst(1.0);
            } else if (id_of("qd", k) >= 0) seed[id_of("qd", k)] = Gen::cst(1.0);
            const std::vector<Sym> T = g.tangent(upto, seed);
            for (int i = 0; i < N; i++) {
                Sym d = Gen::zero();
                if (tau[i].k == Sym::O && !tau[i].x.isc) d = tau[i].x.neg ? g.neg(T[tau[i].x.id]) : T[tau[i].x.id];
                g.code.push_back(assign(g, std::string(dir < N ? "dq[" : "dqd[") + std::to_string(i * N + k) + "]", d));
            }
        }
    } else {
        err = "unknown generator mode";
        return -1;
    }
    return 0;
}

} // namespace

int b2k_rne_generate(const b2k_rne_s *r, const b2k_gen_opts &o, b2k_gen_out &out)
{
    if (o.mode == B2K_GEN_TREE_REGRESSOR) { out.error = "the tree regressor is no operation of DH arms"; return -1; }
    const int N = r->n;
    Gen g;
    std::vector<Link> L(N);
    auto links = [&]() { // the link table, with this function's joint inputs (st, ct, qq) as fresh leaves
        for (int j = 0; j < N; j++) {
            const double *l = r->L[j];
            const double alpha = l[0], A = l[1], theta = l[2], D = l[3], G = l[20];
            const double sa = snap(sin(alpha)), ca = snap(cos(alpha));
            L[j].pris = ((int)l[4] != 0);
            L[j].sa = Gen::cst(sa);
            L[j].ca = Gen::cst(ca);
            Sym d;
            if (L[j].pris) { // the joint variable is the link offset d = q + offset (qq = q + offset in the kernel), theta is fixed
                L[j].st = Gen::cst(snap(sin(theta)));
                L[j].ct = Gen::cst(snap(cos(theta)));
                d = g.var("qq[" + std::to_string(j) + "]");
            } else {
                L[j].st = g.var("st[" + std::to_string(j) + "]");
                L[j].ct = g.var("ct[" + std::to_string(j) + "]");
                d = Gen::cst(D);
            }
            L[j].ps = {Gen::cst(A), g.fix(g.mul(d, Gen::cst(r->mdh ? -sa : sa))), g.fix(g.mul(d, Gen::cst(ca)))};
            L[j].m = l[6];
            for (int k = 0; k < 3; k++) L[j].r[k] = l[7 + k];
            for (int k = 0; k < 9; k++) L[j].I[k] = l[10 + k];
            L[j].c_jm = G * G * l[19];
            L[j].c_b = G * G * l[21];
            L[j].c_tcp = fabs(G) * l[22];
            L[j].c_tcm = fabs(G) * l[23];
        }
    };
    links();
    const RecFn rec = [&](const Inputs &in) { return recursion(g, L, r->mdh != 0, in); };
    auto function = [](const Gen &gg, const char *sig, const std::vector<std::string> &tail) {
        std::string f = std::string("__device__ __forceinline__ void ") + sig + "\n{\n";
        for (const std::string &s : gg.code) f += s + "\n";
        for (const std::string &s : tail) f += s + "\n";
        return f + "}\n";
    };
    std::vector<std::string> tail;
    const char *sig = nullptr;
    std::string src;
    b2k_gen_opts oo = o;
    if (o.mode == B2K_GEN_RNE_DERIV || o.mode == B2K_GEN_ACCEL_DERIV) oo.has_fext = 0; // no tip wrench
    if (o.mode == B2K_GEN_ACCEL_DERIV) {
        // two functions over one constant bank, as for trees: rne_row, the ACCEL row, and rne_deriv_row, the RNE_DERIV row
        // that the kernel evaluates at the solved qdd* with the same gravity
        oo.mode = B2K_GEN_ACCEL;
        if (assemble(g, N, oo, rec, tail, sig, out.error)) return -1;
        src = function(g, sig, tail);
        g.code.clear();
        tail.clear();
        links();
        oo.mode = B2K_GEN_RNE_DERIV;
    }
    if (assemble(g, N, oo, rec, tail, sig, out.error)) return -1;
    out.source = src + function(g, sig, tail);
    out.consts = g.consts;
    if (out.consts.empty()) out.consts.push_back(0.0);
    out.n_mul = g.n_mul; out.n_fma = g.n_fma; out.n_add = g.n_add;
    out.error.clear();
    return 0;
}

// ------------------------------------------------------------------ rigid-body trees (Robot.rne)
// Featherstone's recursion as the reference's Robot.rne runs it (Robot.py:1704-1903) with spatial vectors in
// [linear; angular] order (spatialmath SpatialVelocity / SpatialForce): per joint group j with T_j = C_j J_j(q),
//   v_j = X_j v_p + s_j qd_j            a_j = X_j a_p + s_j qdd_j + v_j x s_j qd_j      (root: a_p = -gravity)
//   f_j = I_j a_j + v_j x* (I_j v_j)    tau_j = s_j . f_j      f_p += X_j^T f_j,        X_j = Ad(T_j^-1)
// written out on 3-vectors and evaluated symbolically: constant rotations with 0 / +-1 entries become permutations,
// zero inertia entries vanish, the root's velocities are one-component.  Reference quirks kept: the motion subspace
// s_j ignores a joint's flip (ET.s, ET.py:592-608), the group inertia is the plain sum of SpatialInertia(m, r) of its
// links without their rotational inertia, torques come out in group order.
namespace {
struct TreeOps {
    Gen &g;
    Vops v;
    explicit TreeOps(Gen &gg) : g(gg), v(gg) {}
    static double snap01(double x)
    {
        const double r = nearbyint(x);
        return (fabs(x - r) < 4e-16 && fabs(r) <= 1.0) ? r : x;
    }
    V3 constR(const double *C, const V3 &u, bool transpose)
    { // Rc u or Rc^T u, Rc = the rotation part of the 3x4 constant
        V3 a = v.fix(u);
        auto e = [&](int i, int j) { return Gen::cst(snap01(transpose ? C[j * 4 + i] : C[i * 4 + j])); };
        auto row = [&](int i) { return g.sum({g.mul(e(i, 0), a.x), g.mul(e(i, 1), a.y), g.mul(e(i, 2), a.z)}); };
        return {row(0), row(1), row(2)};
    }
    V3 jointR(int axis, const Sym &s, const Sym &c, const V3 &u, bool transpose)
    {
        if (axis > 2) return u; // prismatic: no rotation
        V3 a = v.fix(u);
        const Sym sx = transpose ? s : g.neg(s);
        // rotation about axis k mixes the other two components (cyclic order)
        Sym *comp[3] = {&a.x, &a.y, &a.z};
        const int i = (axis + 1) % 3, j = (axis + 2) % 3;
        V3 r = a;
        Sym *out[3] = {&r.x, &r.y, &r.z};
        *out[i] = g.sum({g.mul(c, *comp[i]), g.mul(sx, *comp[j])});
        *out[j] = g.sum({g.mul(g.neg(sx), *comp[i]), g.mul(c, *comp[j])});
        return r;
    }
    V3 mat3(const double *I6, int r0, int c0, const V3 &u)
    { // 3x3 block (rows r0.., cols c0..) of the 6x6 constant times u
        V3 a = v.fix(u);
        auto row = [&](int i) {
            return g.sum({g.mul(Gen::cst(I6[(r0 + i) * 6 + c0]), a.x), g.mul(Gen::cst(I6[(r0 + i) * 6 + c0 + 1]), a.y),
                          g.mul(Gen::cst(I6[(r0 + i) * 6 + c0 + 2]), a.z)});
        };
        return {row(0), row(1), row(2)};
    }
};
} // namespace

int b2k_tree_generate(const b2k_tree_s *t, const b2k_gen_opts &o, b2k_gen_out &out)
{
    if (o.mode == B2K_GEN_RNE_WRENCH) { out.error = "the base wrench is not available for rigid-body trees"; return -1; }
    const int N = t->n;
    Gen g;
    TreeOps T(g);
    Vops &v = T.v;
    std::vector<Sym> st(N), ct(N), qq(N);
    auto joint_inputs = [&]() { // the joint angle / offset arguments of one generated function
        for (int j = 0; j < N; j++) {
            const std::string k = "[" + std::to_string(t->jindex[j]) + "]";
            st[j] = g.var("st" + k); ct[j] = g.var("ct" + k); qq[j] = g.var("qq" + k);
            if (t->flip[j]) { st[j] = g.neg(st[j]); qq[j] = g.neg(qq[j]); } // eta = -q
        }
    };
    joint_inputs();
    auto unit = [&](int axis, const Sym &x) { // x * e_axis
        V3 u = v.zero();
        (axis % 3 == 0 ? u.x : (axis % 3 == 1 ? u.y : u.z)) = x;
        return u;
    };
    // the motion of group j in its own frame from its parent's: angular / linear velocity w, vl and acceleration aw, av
    // (spatial, Featherstone's), and p, the origin of the joint frame in the parent's.  in.qd / in.qdd are indexed like q
    // (jindex); in.grav is a_grav = MINUS the gravity vector (the caller negates), linear part only
    struct Kin { std::vector<V3> w, vl, aw, av, p; };
    auto kin = [&](int j, const Inputs &in, Kin &K) {
        const V3 &agrav = in.grav;
        std::vector<V3> &w = K.w, &vl = K.vl, &aw = K.aw, &av = K.av, &p = K.p;
        const double *C = t->C[j];
        const int ax = t->axis[j];
        const bool rev = ax < 3;
        const Sym &qdj = in.qd[t->jindex[j]], &qddj = in.qdd[t->jindex[j]];
        auto RT = [&](const V3 &u) { return T.jointR(ax, st[j], ct[j], T.constR(C, u, true), true); };
        // p = pc + Rc (e_axis * eta) for a prismatic joint
        const double pc[3] = {C[3], C[7], C[11]};
        p[j] = v.cst(pc);
        if (!rev) p[j] = v.fix(v.add(p[j], T.constR(C, unit(ax, qq[j]), false)));
        const V3 vJw = rev ? unit(ax, qdj) : v.zero(), vJv = rev ? v.zero() : unit(ax, qdj);
        const V3 aJw = rev ? unit(ax, qddj) : v.zero(), aJv = rev ? v.zero() : unit(ax, qddj);
        const int pa = t->parent[j];
        if (pa < 0) {
            w[j] = vJw; vl[j] = vJv;
            aw[j] = aJw;
            av[j] = v.fix(v.add(RT(agrav), aJv));
        } else {
            w[j] = v.fix(v.add(RT(w[pa]), vJw));
            vl[j] = v.fix(v.add(RT(v.cross_acc(w[pa], p[j], &vl[pa])), vJv));
            const V3 wxJw = v.cross_acc(w[j], vJw);
            aw[j] = v.fix(v.add(v.add(RT(aw[pa]), aJw), wxJw));
            const V3 t1 = RT(v.cross_acc(aw[pa], p[j], &av[pa]));
            const V3 t2 = v.cross_acc(w[j], vJv, &aJv);
            const V3 t3 = v.cross_acc(vl[j], vJw, &t2);
            av[j] = v.fix(v.add(t1, t3));
        }
    };
    // one evaluation of the recursion; the torques come out in group order (Robot.py:1890-1899)
    auto rec = [&](const Inputs &in) {
        Kin K{std::vector<V3>(N), std::vector<V3>(N), std::vector<V3>(N), std::vector<V3>(N), std::vector<V3>(N)};
        std::vector<V3> &w = K.w, &vl = K.vl, &aw = K.aw, &av = K.av, &p = K.p;
        std::vector<V3> fl(N), fa(N);
        for (int j = 0; j < N; j++) {
            kin(j, in, K);
            const double *I6 = t->I6[j];
            const V3 hl = v.fix(v.add(T.mat3(I6, 0, 0, vl[j]), T.mat3(I6, 0, 3, w[j])));
            const V3 ha = v.fix(v.add(T.mat3(I6, 3, 0, vl[j]), T.mat3(I6, 3, 3, w[j])));
            const V3 il = v.add(T.mat3(I6, 0, 0, av[j]), T.mat3(I6, 0, 3, aw[j]));
            const V3 ia = v.add(T.mat3(I6, 3, 0, av[j]), T.mat3(I6, 3, 3, aw[j]));
            fl[j] = v.fix(v.cross_acc(w[j], hl, &il));
            const V3 t4 = v.cross_acc(vl[j], hl, &ia);
            fa[j] = v.fix(v.cross_acc(w[j], ha, &t4));
        }
        std::vector<Sym> tau(N);
        for (int j = N - 1; j >= 0; j--) {
            const int ax = t->axis[j];
            const V3 &f = ax < 3 ? fa[j] : fl[j];
            tau[j] = g.fix(ax % 3 == 0 ? f.x : (ax % 3 == 1 ? f.y : f.z));
            const int pa = t->parent[j];
            if (pa >= 0) {
                const double *C = t->C[j];
                auto R = [&](const V3 &u) { return T.constR(C, T.jointR(ax, st[j], ct[j], u, false), false); };
                const V3 Rf = v.fix(R(fl[j]));
                fl[pa] = v.fix(v.add(fl[pa], Rf));
                const V3 Rn = R(fa[j]);
                const V3 pxf = v.cross_acc(p[j], Rf, &Rn);
                fa[pa] = v.fix(v.add(fa[pa], pxf));
            }
        }
        return tau;
    };
    std::string src;
    if (o.mode == B2K_GEN_TREE_REGRESSOR) {
        // The regressor: tau_i = s_i . f_i, and f_i sums the wrenches of group i and of every group below it, carried in by
        // the backward pass.  So Y[i, 10k + c] is joint i's unit twist s carried OUT to group k (the transpose of the
        // backward step: s_l' = R^T (s_l + s_a x p), s_a' = R^T s_a) dotted with group k's wrench f = I a + v x* (I v) for
        // the basis inertia of parameter c.  Written out with A = av + w x vl (the classical acceleration of the origin):
        //   m: s_l . A      h: s_l x aw + w (s_l . w) - s_l (w . w) + A x s_a      Ib: s_a^T Ib aw + (s_a x w)^T Ib w
        // One case per joint row i, each with the forward pass of the groups it needs (the ancestors of i, i and its
        // subtree): the kernel stages and drains Y one joint row at a time, and a forward pass kept live across the rows
        // would not fit the registers.  Rows of other groups are exact zeros.
        Inputs in;
        std::vector<Sym> qdv(N), qddv(N);
        for (int k = 0; k < N; k++) { qdv[k] = g.var("qd[" + std::to_string(k) + "]"); qddv[k] = g.var("qdd[" + std::to_string(k) + "]"); }
        in.qd = qdv; in.qdd = qddv;
        in.grav = {(o.grav_mask & 1) ? g.var("grav[0]") : Gen::zero(), (o.grav_mask & 2) ? g.var("grav[1]") : Gen::zero(),
                   (o.grav_mask & 4) ? g.var("grav[2]") : Gen::zero()};
        auto dot = [&](const V3 &a, const V3 &b) { return g.sum({g.mul(a.x, b.x), g.mul(a.y, b.y), g.mul(a.z, b.z)}); };
        g.code.push_back("    switch (i) {");
        for (int i = 0; i < N; i++) {
            std::vector<bool> below(N, false), need(N, false); // group k is i or hangs below it / its motion is needed
            for (int k = 0; k < N; k++) below[k] = k == i || (t->parent[k] >= 0 && below[t->parent[k]]);
            for (int k = N - 1; k >= 0; k--)
                if (below[k] || need[k]) { need[k] = true; if (t->parent[k] >= 0) need[t->parent[k]] = true; }
            g.code.push_back("    case " + std::to_string(i) + ": {");
            Kin K{std::vector<V3>(N), std::vector<V3>(N), std::vector<V3>(N), std::vector<V3>(N), std::vector<V3>(N)};
            std::vector<V3> sl(N), sa(N);
            for (int k = 0; k < N; k++) {
                if (!below[k]) {
                    if (need[k]) kin(k, in, K);
                    for (int c = 0; c < 10; c++) g.code.push_back("        y[" + std::to_string(10 * k + c) + "] = (real)0;");
                    continue;
                }
                kin(k, in, K);
                const int ax = t->axis[k];
                if (k == i) { // the motion subspace of joint i (ignoring its flip, as rne does)
                    sl[k] = ax < 3 ? v.zero() : unit(ax, Gen::cst(1.0));
                    sa[k] = ax < 3 ? unit(ax, Gen::cst(1.0)) : v.zero();
                } else {
                    const int pa = t->parent[k];
                    const double *C = t->C[k];
                    auto RT = [&](const V3 &u) { return T.jointR(ax, st[k], ct[k], T.constR(C, u, true), true); };
                    sl[k] = v.fix(RT(v.cross_acc(sa[pa], K.p[k], &sl[pa])));
                    sa[k] = v.fix(RT(sa[pa]));
                }
                const V3 &w = K.w[k], &aw = K.aw[k], &s_l = sl[k], &s_a = sa[k];
                const V3 A = v.fix(v.cross_acc(w, K.vl[k], &K.av[k]));
                const Sym slw = g.fix(dot(s_l, w)), ww = g.fix(dot(w, w));
                const V3 hw = v.scale(slw, w), hs = v.scale(g.neg(ww), s_l);
                const V3 t1 = v.cross_acc(A, s_a, &hw, &hs);
                const V3 hcoef = v.cross_acc(s_l, aw, &t1);
                const V3 u = v.fix(v.cross_acc(s_a, w));
                const V3 sa_ = v.fix(s_a), aw_ = v.fix(aw), w_ = v.fix(w);
                auto sum2 = [&](const Sym &a1, const Sym &b1, const Sym &a2, const Sym &b2) { return g.sum({g.mul(a1, b1), g.mul(a2, b2)}); };
                const Sym coef[10] = {dot(s_l, A), hcoef.x, hcoef.y, hcoef.z,
                                      sum2(sa_.x, aw_.x, u.x, w_.x), sum2(sa_.y, aw_.y, u.y, w_.y), sum2(sa_.z, aw_.z, u.z, w_.z),
                                      g.sum({g.mul(sa_.x, aw_.y), g.mul(sa_.y, aw_.x), g.mul(u.x, w_.y), g.mul(u.y, w_.x)}),
                                      g.sum({g.mul(sa_.y, aw_.z), g.mul(sa_.z, aw_.y), g.mul(u.y, w_.z), g.mul(u.z, w_.y)}),
                                      g.sum({g.mul(sa_.x, aw_.z), g.mul(sa_.z, aw_.x), g.mul(u.x, w_.z), g.mul(u.z, w_.x)})};
                for (int c = 0; c < 10; c++) g.code.push_back("    " + assign(g, "y[" + std::to_string(10 * k + c) + "]", coef[c]));
            }
            g.code.push_back("    } break;");
        }
        g.code.push_back("    }");
        src = "__device__ __forceinline__ void rne_regressor_row(const real *C, const real *grav, const real *fext, const real *st, "
              "const real *ct, const real *qq, const real *qd, const real *qdd, int i, real *y)\n{\n";
        for (const std::string &s : g.code) src += s + "\n";
        src += "}\n";
        out.source = src;
        out.consts = g.consts;
        if (out.consts.empty()) out.consts.push_back(0.0);
        out.n_mul = g.n_mul; out.n_fma = g.n_fma; out.n_add = g.n_add;
        out.error.clear();
        return 0;
    }
    std::vector<std::string> tail;
    const char *sig = nullptr;
    b2k_gen_opts oo = o;
    oo.has_fext = 0; // Robot.rne has no tip wrench
    if (o.mode == B2K_GEN_ACCEL_DERIV) {
        // two functions over one constant bank: rne_row, the ACCEL row (M and torque - rne(q, qd, 0)), and rne_deriv_row,
        // the RNE_DERIV row that the kernel evaluates at the solved qdd* with the same gravity
        oo.mode = B2K_GEN_ACCEL;
        if (assemble(g, N, oo, rec, tail, sig, out.error)) return -1;
        src = std::string("__device__ __forceinline__ void ") + sig + "\n{\n";
        for (const std::string &s : g.code) src += s + "\n";
        for (const std::string &s : tail) src += s + "\n";
        src += "}\n";
        g.code.clear();
        tail.clear();
        joint_inputs();
        oo.mode = B2K_GEN_RNE_DERIV;
    }
    if (assemble(g, N, oo, rec, tail, sig, out.error)) return -1;
    src += std::string("__device__ __forceinline__ void ") + sig + "\n{\n";
    for (const std::string &s : g.code) src += s + "\n";
    for (const std::string &s : tail) src += s + "\n";
    src += "}\n";
    out.source = src;
    out.consts = g.consts;
    if (out.consts.empty()) out.consts.push_back(0.0);
    out.n_mul = g.n_mul; out.n_fma = g.n_fma; out.n_add = g.n_add;
    out.error.clear();
    return 0;
}
