// Partial evaluation of a template's `violation` rule against concrete parameters -> formula tree, and
// formula tree -> jump-threaded instructions.  See lower.hpp for the scheme.
#include <cmath>
#include "lower.hpp"

#include <algorithm>
#include <cstring>
#include <functional>
#include <set>

namespace gk {

// ====================================================================================== formulas
static FP mk(Formula::K k) {
  auto f = std::make_shared<Formula>();
  f->k = k;
  return f;
}
FP f_true() {
  static FP t = mk(Formula::True);
  return t;
}
FP f_false() {
  static FP f = mk(Formula::False);
  return f;
}
FP f_and(FP a, FP b) {
  if (a->k == Formula::False || b->k == Formula::False) return f_false();
  if (a->k == Formula::True) return b;
  if (b->k == Formula::True) return a;
  auto f = std::make_shared<Formula>();
  f->k = Formula::And;
  if (a->k == Formula::And) f->kids = a->kids;
  else f->kids.push_back(a);
  if (b->k == Formula::And) f->kids.insert(f->kids.end(), b->kids.begin(), b->kids.end());
  else f->kids.push_back(b);
  return f;
}
FP f_or(FP a, FP b) {
  if (a->k == Formula::True || b->k == Formula::True) return f_true();
  if (a->k == Formula::False) return b;
  if (b->k == Formula::False) return a;
  auto f = std::make_shared<Formula>();
  f->k = Formula::Or;
  if (a->k == Formula::Or) f->kids = a->kids;
  else f->kids.push_back(a);
  if (b->k == Formula::Or) f->kids.insert(f->kids.end(), b->kids.begin(), b->kids.end());
  else f->kids.push_back(b);
  return f;
}
FP f_not(FP a) {
  if (a->k == Formula::True) return f_false();
  if (a->k == Formula::False) return f_true();
  if (a->k == Formula::Not) return a->kids[0];
  auto f = std::make_shared<Formula>();
  f->k = Formula::Not;
  f->kids.push_back(a);
  return f;
}
FP f_exists(int scope, FP body) {
  if (body->k == Formula::False) return f_false();
  auto f = std::make_shared<Formula>();
  f->k = Formula::Exists;
  f->scope = scope;
  f->kids.push_back(body);
  return f;
}
FP f_exists2(int scope, FP body) {
  if (body->k == Formula::False) return f_false();
  auto f = std::make_shared<Formula>();
  f->k = Formula::Exists;
  f->scope = scope;
  f->two = true;
  f->kids.push_back(body);
  return f;
}
static FP f_atom(int op, int col, VP cval = nullptr, uint32_t imm = 0) {
  auto f = std::make_shared<Formula>();
  f->k = Formula::Atom;
  f->op = op;
  f->col = col;
  f->cval = std::move(cval);
  f->imm = imm;
  return f;
}
size_t formula_size(const FP& f) {
  size_t n = 1;
  for (auto& k : f->kids) n += formula_size(k);
  return n;
}
std::string formula_str(const FP& f, const Schema& s) {
  switch (f->k) {
    case Formula::True: return "T";
    case Formula::False: return "F";
    case Formula::Not: return "!" + formula_str(f->kids[0], s);
    case Formula::And:
    case Formula::Or: {
      std::string o = "(";
      for (size_t i = 0; i < f->kids.size(); ++i) {
        if (i) o += f->k == Formula::And ? " & " : " | ";
        o += formula_str(f->kids[i], s);
      }
      return o + ")";
    }
    case Formula::Exists: return std::string(f->two ? "E2[s" : "E[s") + std::to_string(f->scope) + ":" + s.scopes[f->scope].gen->key + "]{" + formula_str(f->kids[0], s) + "}";
    case Formula::Atom: {
      static const char* names[] = {"?", "truthy", "defined", "vtmask", "sid_eq", "sid_in", "num_cmp", "prefix", "suffix",
                                    "contains", "anyprefix", "anysuffix"};
      std::string o = std::string(names[f->op]) + "(" + s.cols[f->col].expr->key;
      if (f->cval) o += ", " + fmt_value(f->cval, false);
      if (f->op == GK_OP_NUM_CMP || f->op == GK_OP_VTMASK) o += ", #" + std::to_string(f->imm);
      return o + ")";
    }
  }
  return "?";
}

// ====================================================================================== schema
// ====================================================================================== device-evaluable closures
struct RawArg {
  CP base;
  std::vector<VP> keys;
};
// Walks a closure's term: false unless it is a closed pure term (no `input` / `data`, no impure rule); collects the
// `<captured column>[literal keys...]` paths it reads.
static bool lut_args(const Module& m, const Term* t, const Closure& c, std::vector<RawArg>& out) {
  if (!t) return true;
  auto cap_of = [&](int vid) -> const CapArg* {
    for (auto& cp : c.caps)
      if (cp.first == vid) return &cp.second;
    return nullptr;
  };
  if (t->k == TK::Var) {
    if (t->vid == m.vid_input || t->vid == m.vid_data) return false;
    if (const CapArg* cap = cap_of(t->vid)) {
      if (cap->k == CapArg::Col) out.push_back(RawArg{cap->col, {}});
      return true;
    }
    if (m.is_rule(t->name)) return false;      // a (non-function) rule used as a value
    return true;                                // a local of a comprehension / wildcard
  }
  if (t->k == TK::Ref && t->head->k == TK::Var) {
    const CapArg* cap = cap_of(t->head->vid);
    if (cap && cap->k == CapArg::Col) {
      std::vector<VP> keys;
      size_t i = 0;
      for (; i < t->args.size() && t->args[i]->k == TK::Scalar; ++i) keys.push_back(t->args[i]->val);
      out.push_back(RawArg{cap->col, std::move(keys)});
      for (; i < t->args.size(); ++i)
        if (!lut_args(m, t->args[i].get(), c, out)) return false;
      return true;
    }
  }
  if (t->k == TK::Call && m.is_rule(t->name)) {
    auto pf = m.pure_fn.find(t->name);
    if (pf == m.pure_fn.end() || !pf->second) return false;
  }
  if (t->head && !lut_args(m, t->head.get(), c, out)) return false;
  for (auto& a : t->args)
    if (!lut_args(m, a.get(), c, out)) return false;
  for (auto& kv : t->kvs)
    if (!lut_args(m, kv.first.get(), c, out) || !lut_args(m, kv.second.get(), c, out)) return false;
  if (!lut_args(m, t->key.get(), c, out) || !lut_args(m, t->value.get(), c, out)) return false;
  for (auto& s2 : t->body)
    if (!lut_args(m, s2.a.get(), c, out) || !lut_args(m, s2.b.get(), c, out) || !lut_args(m, s2.c.get(), c, out)) return false;
  return true;
}

static void add_leaf(std::vector<XInfo::Arg>& out, const CP& leaf, const std::vector<VP>& keys) {
  for (auto& a : out)
    if (a.leaf.get() == leaf.get() && (!leaf || true) && a.keys.size() == keys.size()) {
      bool same = (a.leaf && leaf) ? a.leaf->key == leaf->key : (!a.leaf && !leaf);
      for (size_t i = 0; i < keys.size() && same; ++i) same = v_eq(a.keys[i], keys[i]);
      if (same) return;
    }
  out.push_back(XInfo::Arg{leaf, keys});
}
// the leaf values behind  <base>[keys...]  (false: something on the way needs the host)
static bool leaf_args_of(const CP& base, const std::vector<VP>& keys, std::vector<XInfo::Arg>& out) {
  const XInfo bi = closure_xinfo(*base);
  switch (bi.k) {
    case XK::Elem:
    case XK::Key: add_leaf(out, base, keys); return true;
    case XK::Path: {
      std::vector<VP> all = bi.keys;
      all.insert(all.end(), keys.begin(), keys.end());
      if (bi.from_input) {
        add_leaf(out, nullptr, all);
        return true;
      }
      return leaf_args_of(bi.base, all, out);
    }
    case XK::Count:
    case XK::Lut:
      for (auto& a : bi.args) add_leaf(out, a.leaf, a.keys);   // (the keys index the COMPUTED value, not a leaf)
      return true;
    default: return false;
  }
}
static bool leafy_arg(const XInfo::Arg& a) {
  // may this value be (part of) a lookup key?  A whole iterated element, the whole object or its `spec` are not: every
  // object would be its own key and the host would evaluate the closure once per object again
  if (!a.leaf) return a.keys.size() >= 4;                       // review.object.<x>.<y>...
  if (a.leaf->leaf == Closure::Key) return true;
  return !a.keys.empty();
}

bool xinfo_leaf_args(const CP& base, const std::vector<VP>& keys, std::vector<XInfo::Arg>& out) { return leaf_args_of(base, keys, out); }

XInfo closure_xinfo(const Closure& c) {
  XInfo x;
  if (c.leaf == Closure::Elem) {
    x.k = XK::Elem;
    return x;
  }
  if (c.leaf == Closure::Key) {
    x.k = XK::Key;
    return x;
  }
  if (!c.term || !c.mod) return x;
  const Term& t = *c.term;
  const Module& m = *c.mod;
  auto cap_of = [&](int vid) -> const CapArg* {
    for (auto& cp : c.caps)
      if (cp.first == vid) return &cp.second;
    return nullptr;
  };
  if (t.k == TK::Ref && t.head->k == TK::Var) {
    bool lit = true;
    for (auto& a : t.args) lit = lit && a->k == TK::Scalar;
    const CapArg* cap = cap_of(t.head->vid);
    if (lit && cap && cap->k == CapArg::Col) {
      const XK bk = closure_xinfo(*cap->col).k;
      if (bk == XK::Path || bk == XK::Elem || bk == XK::Key) {
        x.k = XK::Path;
        x.base = cap->col;
        for (auto& a : t.args) x.keys.push_back(a->val);
        return x;
      }
    }
    if (lit && !cap && t.head->vid == m.vid_input && !t.args.empty() && t.args[0]->val->t == VT::Str && t.args[0]->val->s == "review") {
      x.k = XK::Path;
      x.from_input = true;
      for (auto& a : t.args) x.keys.push_back(a->val);
      return x;
    }
  }
  if (t.k == TK::Call && t.name == "count" && !m.is_rule(t.name) && t.args.size() == 1 && t.args[0]->k == TK::Var) {
    const CapArg* cap = cap_of(t.args[0]->vid);
    if (cap && cap->k == CapArg::Col) {
      const XK bk = closure_xinfo(*cap->col).k;
      if (bk == XK::Path || bk == XK::Elem) {
        x.k = XK::Count;
        x.base = cap->col;
        if (!leaf_args_of(cap->col, {}, x.args)) return XInfo();
        return x;
      }
    }
  }
  std::vector<RawArg> raw;
  if (!lut_args(m, &t, c, raw)) return XInfo();
  for (auto& r : raw)
    if (!leaf_args_of(r.base, r.keys, x.args)) return XInfo();
  for (auto& a : x.args)
    if (!leafy_arg(a)) return XInfo();
  if (x.args.empty() || x.args.size() > 4) return XInfo();
  x.k = XK::Lut;
  return x;
}

bool schema_device_ingestable(const Schema& s, std::string* why) {
  for (size_t i = 1; i < s.scopes.size(); ++i) {
    const XK k = closure_xinfo(*s.scopes[i].gen).k;
    if (k != XK::Path && k != XK::Elem) {
      if (why) *why = "scope generator " + s.scopes[i].gen->key;
      return false;
    }
  }
  for (auto& c : s.cols)
    if (closure_xinfo(*c.expr).k == XK::Host) {
      if (why) *why = "column " + c.expr->key;
      return false;
    }
  return true;
}

[[noreturn]] static void not_on_device(const std::string& key) {
  throw RegoError{"rego_unsupported: device-ingest: the ingest kernels cannot compute " + key};
}

int Schema::scope_for(const CP& gen) {
  auto it = scope_ix.find(gen->key);
  if (it != scope_ix.end()) return it->second;
  if (device_only) {
    const XK k = closure_xinfo(*gen).k;
    if (k != XK::Path && k != XK::Elem) not_on_device(gen->key);
  }
  ScopeDef d;
  d.parent = gen->scope;
  d.gen = gen;
  d.depth = scopes[gen->scope].depth + 1;
  if (d.depth > GK_MAX_LOOP_DEPTH) throw RegoError{"rego_unsupported: iteration nesting deeper than " + std::to_string(GK_MAX_LOOP_DEPTH)};
  scopes.push_back(d);
  int id = (int)scopes.size() - 1;
  scope_ix[gen->key] = id;
  return id;
}
int Schema::col_for(const CP& expr, uint32_t enc) {
  auto it = col_ix.find(expr->key);
  if (it != col_ix.end()) {
    cols[it->second].enc |= enc;
    return it->second;
  }
  if (device_only && closure_xinfo(*expr).k == XK::Host) not_on_device(expr->key);
  ColDef d;
  d.expr = expr;
  d.scope = expr->scope;
  d.enc = enc;
  cols.push_back(d);
  int id = (int)cols.size() - 1;
  if (id >= 65535) throw RegoError{"rego_unsupported: too many feature columns"};
  col_ix[expr->key] = id;
  return id;
}

// ====================================================================================== lowering
namespace {

struct SymVal {
  enum K : uint8_t { Conc, Col, Bool, Arr, ObjLit, Opaque, DiffCS, DiffSC, Count, SetOf, ArrHoles } k = Conc;
  VP v;                                                   // Conc; DiffCS/DiffSC: the concrete set
  CP col;                                                 // Col
  std::shared_ptr<SymVal> sym;                            // DiffCS/DiffSC: the symbolic collection (Col or SetOf)
  // SetOf / ArrHoles: `f` is a formula with holes (Atom op == -1, imm == j); items[j].second is the head produced at hole j.
  // ArrHoles is an array comprehension that iterates an OBJECT collection while mixing in parameters: its length is not
  // known at lowering time, so only the existential consumers take it -- any(), all(), count() against 0.
  // The set is { head_j | path condition of hole j }.
  FP f;                                                   // Bool: value; Opaque: definedness
  FP d;                                                   // Bool: definedness of the value (null: always defined).  `f` decides statements
                                                          // (`x`, `not x`); `d` matters where an undefined value differs from a false one:
                                                          // `y := x`, comprehension heads, count(), all(), `x == false`
  bool compr = false;                                     // Arr: built by a comprehension (undefined heads are absent), not a literal
  std::vector<std::pair<FP, SymVal>> items;               // Arr: (guard, element); Count: [0] = counted value
  std::vector<std::pair<VP, SymVal>> fields;              // ObjLit
  bool tainted = false;                                   // Conc: derived from input.parameters
  bool row_dep = false;                                   // Opaque: built from a value of an iteration that was open at that point
  static SymVal conc(VP v, bool tainted = false) { SymVal s; s.k = Conc; s.v = std::move(v); s.tainted = tainted; return s; }
  static SymVal column(CP c) { SymVal s; s.k = Col; s.col = std::move(c); return s; }
  static SymVal boolean(FP f, FP d = nullptr) { SymVal s; s.k = Bool; s.f = std::move(f); s.d = std::move(d); return s; }
  static SymVal opaque(FP def) { SymVal s; s.k = Opaque; s.f = std::move(def); return s; }
};

struct LEnv {
  std::vector<std::pair<int, SymVal>> b;
  const SymVal* find(int vid) const {
    for (size_t i = b.size(); i-- > 0;)
      if (b[i].first == vid) return &b[i].second;
    return nullptr;
  }
  size_t mark() const { return b.size(); }
  void undo(size_t m) { b.resize(m); }
  void bind(int vid, SymVal v) { b.emplace_back(vid, std::move(v)); }
};

struct Deps {
  bool obj = false, param = false, iter = false, mixed = false;
  bool data = false;   // reads data.inventory, directly or through a captured column
  void operator|=(const Deps& o) {
    data |= o.data;
    obj |= o.obj;
    param |= o.param;
    iter |= o.iter;
    mixed |= o.mixed;
  }
};

[[noreturn]] void unsupported(const std::string& what, int line) {
  throw RegoError{"rego_unsupported: " + what + " (line " + std::to_string(line) + ") cannot be lowered to the GPU predicate table"};
}

using BodyK = std::function<FP(LEnv&)>;
using SymK = std::function<FP(const SymVal&)>;

class Lowerer {
 public:
  Lowerer(std::shared_ptr<const Module> mod, VP params, Schema& schema)
      : mod_(std::move(mod)), m_(*mod_), schema_(schema), params_(params),
        ev_(m_, v_obj({{v_str("parameters"), params}})) {
    vid_cur_ = const_cast<Module&>(m_).intern("$cur");
    vid_key_ = const_cast<Module&>(m_).intern("$key");
  }

  bool product_mode = false;

  FP run() {
    auto it = m_.rules.find("violation");
    if (it == m_.rules.end()) throw RegoError{"rego_compile_error: template has no `violation` rule"};
    FP out = f_false();
    head_paths_ = 0;
    head_object_level_ = true;
    for (auto& r : it->second) {
      if (r.kind != Rule::PSet) throw RegoError{"rego_type_error: `violation` must be a partial set rule"};
      LEnv env;
      FP f = lower_body(r.body, 0, env, [&](LEnv& e) {
        // how many results one (constraint, object) pair can have: the head is reached along `head_paths_` lowering paths; if
        // that is one and the head names only parameters and object-level values, the set has at most ONE element
        ++head_paths_;
        head_object_level_ = head_object_level_ && object_level_term(r.key, e);
        // every arrival at the head is marked with a hole of its own: distinct paths never merge, and the ambiguity formula
        // below can tell which parts of the predicate a result's bindings come from
        return sym_term(r.key, e, [&](const SymVal& kv) {
          auto h = std::make_shared<Formula>();
          h->k = Formula::Atom;
          h->op = -1;
          h->imm = (uint32_t)nholes_++;
          return f_and(defined_cond(kv), FP(h));
        });
      });
      out = f_or(out, f);
      check_size(out, r.line);
    }
    const auto plug = [](uint32_t) { return f_true(); };
    has_hole_.clear();
    amb_ = fill_tree(amb_of(out), plug);
    if (formula_size(amb_) > 40000) amb_ = f_true();
    return fill_tree(out, plug);
  }
  FP ambiguity() const { return amb_; }

  // May the pair have more than one result?  Only the parts of the predicate that hold a head (a hole) bind what a result is made
  // of: two of them true together, or an iteration around a head with two satisfying rows.  Hole-free parts are plain conditions.
  bool has_hole(const FP& f) {
    auto it = has_hole_.find(f.get());
    if (it != has_hole_.end()) return it->second;
    bool h = f->k == Formula::Atom && f->op == -1;
    for (auto& k : f->kids) h = has_hole(k) || h;
    has_hole_.emplace(f.get(), h);
    return h;
  }
  FP amb_of(const FP& f) {
    if (!has_hole(f)) return f_false();
    switch (f->k) {
      case Formula::And: {
        FP any = f_false();
        for (auto& k : f->kids) any = f_or(any, amb_of(k));
        return any->k == Formula::False ? any : f_and(f, any);
      }
      case Formula::Or: {
        FP any = f_false(), two = f_false(), later = f_false();
        for (size_t i = f->kids.size(); i-- > 0;) {
          const FP& k = f->kids[i];
          any = f_or(any, amb_of(k));
          if (!has_hole(k)) continue;
          two = f_or(two, f_and(k, later));   // this one and a later one
          later = f_or(later, k);
        }
        return f_or(any, two);
      }
      case Formula::Exists: return f_or(f_exists2(f->scope, f->kids[0]), f_exists(f->scope, amb_of(f->kids[0])));
      default: return f_false();   // a hole itself; (a head never sits under a negation)
    }
  }

  // at most one result per (constraint, object): audit totals can take the pair count (pkg/audit/manager.go:886-945 counts results)
  bool single_result() const { return head_paths_ <= 1 && head_object_level_; }

  // does the value read a column of a scope that is OPEN where the head is evaluated (a per-row value)?  Values aggregated over
  // a closed iteration (comprehensions, count(), set differences) are one value per object.
  bool scope_open(int scope) const { return scope != 0 && std::find(iter_stack_.begin(), iter_stack_.end(), scope) != iter_stack_.end(); }
  bool formula_reads_open(const FP& f) const {
    if (!f) return false;
    if (f->k == Formula::Atom) return f->col >= 0 && scope_open(schema_.cols[f->col].scope);
    for (auto& k : f->kids)
      if (formula_reads_open(k)) return true;
    return false;
  }
  bool object_level_val(const SymVal& s) const {
    if (s.row_dep) return false;
    if (s.k == SymVal::Col && scope_open(s.col->scope)) return false;
    if (formula_reads_open(s.f) || formula_reads_open(s.d)) return false;
    if (s.sym && !object_level_val(*s.sym)) return false;
    for (auto& it : s.items)
      if (formula_reads_open(it.first) || !object_level_val(it.second)) return false;
    for (auto& f : s.fields)
      if (!object_level_val(f.second)) return false;
    return true;
  }
  bool object_level_term(const TP& t, LEnv& env) {
    Deps d = deps(t, env, false);
    if (d.iter) return false;   // the head itself iterates
    std::vector<int> fv;
    free_vars(t, fv);
    for (int v : fv)
      if (const SymVal* sv = env.find(v))
        if (!object_level_val(*sv)) return false;
    return true;
  }

 private:
  std::shared_ptr<const Module> mod_;
  const Module& m_;
  Schema& schema_;
  VP params_;
  Eval ev_;
  int vid_cur_, vid_key_;
  int depth_ = 0;
  int head_paths_ = 0;
  bool head_object_level_ = true;
  int nholes_ = 0;
  FP amb_;
  std::unordered_map<const Formula*, bool> has_hole_;
  std::map<std::string, Deps> rule_deps_;
  std::set<std::string> rule_deps_busy_;
  std::vector<std::shared_ptr<Term>> synth_;   // keeps synthesized terms alive

  void check_size(const FP& f, int line) {
    if (formula_size(f) > 20000) unsupported("predicate too large after partial evaluation", line);
  }

  // ------------------------------------------------------------------ dependency classification
  bool unbound(const Term& t, const LEnv& env) const {
    return t.k == TK::Var && !env.find(t.vid) && t.vid != m_.vid_input && t.vid != m_.vid_data && !m_.is_rule(t.name);
  }

  Deps rule_deps(const std::string& name) {
    auto it = rule_deps_.find(name);
    if (it != rule_deps_.end()) return it->second;
    if (rule_deps_busy_.count(name)) return Deps();
    rule_deps_busy_.insert(name);
    Deps d;
    LEnv empty;
    for (auto& r : m_.rules.at(name)) {
      if (r.key) d |= deps(r.key, empty, true);
      if (r.value) d |= deps(r.value, empty, true);
      d |= body_deps(r.body, empty);
      for (auto& el : r.els) {
        if (el.first) d |= deps(el.first, empty, true);
        d |= body_deps(el.second, empty);
      }
    }
    d.iter = false;
    rule_deps_busy_.erase(name);
    rule_deps_[name] = d;
    return d;
  }

  Deps body_deps(const std::vector<Stmt>& body, const LEnv& env) {
    Deps d;
    for (auto& s : body) {
      if (s.a) d |= deps(s.a, env, true);
      if (s.b) d |= deps(s.b, env, true);
      if (s.c) d |= deps(s.c, env, true);
    }
    return d;
  }

  // `local`: unbound variables are comprehension/function locals, not iteration at this level
  Deps deps(const TP& t, const LEnv& env, bool local) {
    Deps d;
    switch (t->k) {
      case TK::Scalar: break;
      case TK::Var: {
        if (const SymVal* s = env.find(t->vid)) {
          if (s->k == SymVal::Col) d.obj = true, d.data = d.data || s->col->uses_data;
          else if (s->k != SymVal::Conc) d.mixed = d.obj = d.param = true;
          else if (s->tainted) d.param = true;
        } else if (t->vid == m_.vid_input) {
          d.obj = d.param = true;
        } else if (t->vid == m_.vid_data) {
          // data.inventory (referential constraints): varies with the synced cache, not with the constraint -- object-side, never folded
          d.obj = d.data = true;
          schema_.uses_data = true;
        } else if (m_.is_rule(t->name)) {
          d |= rule_deps(t->name);
        } else if (!local) {
          d.iter = true;
        }
        break;
      }
      case TK::Ref: {
        size_t start = 0;
        if (t->head->k == TK::Var && t->head->vid == m_.vid_input && !env.find(t->head->vid) && !t->args.empty() &&
            t->args[0]->k == TK::Scalar && t->args[0]->val->t == VT::Str) {
          const std::string& f = t->args[0]->val->s;
          if (f == "parameters") d.param = true;
          else if (f == "review") d.obj = true;
          else d.obj = d.param = true;
          start = 1;
        } else {
          d |= deps(t->head, env, local);
        }
        for (size_t i = start; i < t->args.size(); ++i) d |= deps(t->args[i], env, local);
        break;
      }
      case TK::Call: {
        auto it = m_.rules.find(t->name);
        if (it != m_.rules.end()) d |= rule_deps(t->name);
        else if (!is_builtin(t->name)) throw RegoError{"rego_type_error: undefined function " + t->name + " (line " + std::to_string(t->line) + ")"};
        for (auto& a : t->args) d |= deps(a, env, local);
        break;
      }
      case TK::Array:
      case TK::Set:
        for (auto& a : t->args) d |= deps(a, env, local);
        break;
      case TK::Object:
        for (auto& kv : t->kvs) {
          d |= deps(kv.first, env, local);
          d |= deps(kv.second, env, local);
        }
        break;
      case TK::ArrCompr:
      case TK::SetCompr:
      case TK::ObjCompr: {
        Deps x;
        if (t->key) x |= deps(t->key, env, true);
        x |= deps(t->value, env, true);
        x |= body_deps(t->body, env);
        x.iter = false;
        d |= x;
        break;
      }
    }
    return d;
  }

  static bool pure_conc(const Deps& d) { return !d.obj && !d.mixed; }
  static bool pure_obj(const Deps& d) { return d.obj && !d.param && !d.mixed && !d.iter; }

  // ------------------------------------------------------------------ closures
  void free_vars(const TP& t, std::vector<int>& out) const {
    if (!t) return;
    if (t->k == TK::Var) out.push_back(t->vid);
    if (t->head) free_vars(t->head, out);
    for (auto& a : t->args) free_vars(a, out);
    for (auto& kv : t->kvs) {
      free_vars(kv.first, out);
      free_vars(kv.second, out);
    }
    free_vars(t->key, out);
    free_vars(t->value, out);
    for (auto& s : t->body) {
      free_vars(s.a, out);
      free_vars(s.b, out);
      free_vars(s.c, out);
    }
  }

  bool refs_module(const TP& t) const {
    if (!t) return false;
    if (t->k == TK::Var && m_.is_rule(t->name)) return true;
    if (t->k == TK::Call && m_.is_rule(t->name)) return true;
    if (t->head && refs_module(t->head)) return true;
    for (auto& a : t->args)
      if (refs_module(a)) return true;
    for (auto& kv : t->kvs)
      if (refs_module(kv.first) || refs_module(kv.second)) return true;
    if (refs_module(t->key) || refs_module(t->value)) return true;
    for (auto& s : t->body)
      if (refs_module(s.a) || refs_module(s.b) || refs_module(s.c)) return true;
    return false;
  }

  static void subst_print(const Term& t, const std::map<int, std::string>& sub, std::string& out);

  void collect_rule_refs(const TP& t, std::set<std::string>& out) const {
    if (!t) return;
    if ((t->k == TK::Var || t->k == TK::Call) && m_.is_rule(t->name) && out.insert(t->name).second) {
      for (auto& r : m_.rules.at(t->name)) {
        for (auto& a : r.args) collect_rule_refs(a, out);
        collect_rule_refs(r.key, out);
        collect_rule_refs(r.value, out);
        for (auto& s : r.body) {
          collect_rule_refs(s.a, out);
          collect_rule_refs(s.b, out);
          collect_rule_refs(s.c, out);
        }
        for (auto& e : r.els) {
          collect_rule_refs(e.first, out);
          for (auto& s : e.second) {
            collect_rule_refs(s.a, out);
            collect_rule_refs(s.b, out);
            collect_rule_refs(s.c, out);
          }
        }
      }
    }
    if (t->head) collect_rule_refs(t->head, out);
    for (auto& a : t->args) collect_rule_refs(a, out);
    for (auto& kv : t->kvs) {
      collect_rule_refs(kv.first, out);
      collect_rule_refs(kv.second, out);
    }
    collect_rule_refs(t->key, out);
    collect_rule_refs(t->value, out);
    for (auto& s : t->body) {
      collect_rule_refs(s.a, out);
      collect_rule_refs(s.b, out);
      collect_rule_refs(s.c, out);
    }
  }
  std::string rules_signature(const TP& t) const {
    std::set<std::string> names;
    collect_rule_refs(t, names);
    std::string text;
    for (auto& n : names) text += rule_str(m_, n);
    // FNV-1a 64
    uint64_t h = 1469598103934665603ull;
    for (unsigned char ch : text) {
      h ^= ch;
      h *= 1099511628211ull;
    }
    char buf[24];
    snprintf(buf, sizeof buf, "%016llx", (unsigned long long)h);
    return buf;
  }

  bool touches_data(const TP& t) const {
    if (!t) return false;
    if (t->k == TK::Var && t->vid == m_.vid_data) return true;
    if (touches_data(t->head) || touches_data(t->key) || touches_data(t->value)) return true;
    for (auto& a : t->args)
      if (touches_data(a)) return true;
    for (auto& kv : t->kvs)
      if (touches_data(kv.first) || touches_data(kv.second)) return true;
    for (auto& st : t->body)
      if (touches_data(st.a) || touches_data(st.b) || touches_data(st.c)) return true;
    if (t->k == TK::Call && m_.is_rule(t->name)) {   // a helper function that reads data.inventory itself
      bool doc = false;
      std::vector<std::string> refs;
      (void)refs;
      auto it = m_.rules.find(t->name);
      if (it != m_.rules.end())
        for (auto& r : it->second) {
          for (auto& st : r.body)
            if (touches_data(st.a) || touches_data(st.b) || touches_data(st.c)) doc = true;
          if (touches_data(r.value) || touches_data(r.key)) doc = true;
        }
      return doc;
    }
    return false;
  }
  // every variable of the term that the environment binds is a constant or a column: the term can become a closure with the
  // constants captured (and it names no parameter directly)
  bool closable(const TP& term, const LEnv& env) {
    std::vector<int> fv;
    free_vars(term, fv);
    for (int v : fv) {
      const SymVal* sv = env.find(v);
      if (sv && sv->k != SymVal::Conc && sv->k != SymVal::Col) return false;
    }
    return !names_parameters(term);
  }
  bool names_parameters(const TP& t) const {
    if (!t) return false;
    if (t->k == TK::Var && t->vid == m_.vid_input) return true;   // a bare `input`
    if (t->k == TK::Ref && t->head && t->head->k == TK::Var && t->head->vid == m_.vid_input) {
      if (t->args.empty() || t->args[0]->k != TK::Scalar || t->args[0]->val->t != VT::Str || t->args[0]->val->s != "review") return true;
      for (size_t i = 1; i < t->args.size(); ++i)
        if (names_parameters(t->args[i])) return true;
      return false;
    }
    if (names_parameters(t->head) || names_parameters(t->key) || names_parameters(t->value)) return true;
    for (auto& a : t->args)
      if (names_parameters(a)) return true;
    for (auto& kv : t->kvs)
      if (names_parameters(kv.first) || names_parameters(kv.second)) return true;
    for (auto& st : t->body)
      if (names_parameters(st.a) || names_parameters(st.b) || names_parameters(st.c)) return true;
    return false;
  }
  CP make_closure(const TP& term, const LEnv& env) {
    // <path closure>["a"]["b"] is the same column as the longer path from the root: `spec := input.review.object.spec;
    // spec.containers` and `input.review.object.spec.containers` must not become two scopes / two sets of columns
    if (term->k == TK::Ref && term->head->k == TK::Var) {
      bool lit = true;
      for (auto& a : term->args) lit = lit && a->k == TK::Scalar;
      const SymVal* s = env.find(term->head->vid);
      if (lit && s && s->k == SymVal::Col && s->col->leaf == Closure::None && s->col->mod == mod_ && s->col->term->k == TK::Ref &&
          s->col->term->head->k == TK::Var) {
        const Term& bt = *s->col->term;
        bool blit = true;
        for (auto& a : bt.args) blit = blit && a->k == TK::Scalar;
        if (blit) {
          std::vector<TP> path(bt.args.begin(), bt.args.end());
          path.insert(path.end(), term->args.begin(), term->args.end());
          LEnv be;
          for (auto& cp : s->col->caps) be.bind(cp.first, cp.second.k == CapArg::Conc ? SymVal::conc(cp.second.v) : SymVal::column(cp.second.col));
          return make_closure(synth_ref(bt.head, std::move(path), term->line), be);
        }
      }
    }
    auto c = std::make_shared<Closure>();
    c->mod = mod_;
    c->term = term;
    std::vector<int> fv;
    free_vars(term, fv);
    std::sort(fv.begin(), fv.end());
    fv.erase(std::unique(fv.begin(), fv.end()), fv.end());
    std::map<int, std::string> sub;
    int scope = 0;
    for (int v : fv) {
      const SymVal* s = env.find(v);
      if (!s) continue;
      CapArg a;
      if (s->k == SymVal::Conc) {
        a.k = CapArg::Conc;
        a.v = s->v;
        // scalars print as literals so that `spec[field]` with field = "containers" and `spec.containers` are one column
        sub[v] = (s->v->t == VT::Str || s->v->t == VT::Num || s->v->t == VT::True || s->v->t == VT::False || s->v->t == VT::Null)
                     ? fmt_value(s->v, false)
                     : "<" + intern_key(s->v) + ">";
      } else if (s->k == SymVal::Col) {
        a.k = CapArg::Col;
        a.col = s->col;
        sub[v] = "<" + s->col->key + ">";
        int sc = s->col->scope;
        if (sc != scope) {
          // scopes must lie on one ancestor chain; keep the deeper one
          int deep = schema_.scopes[sc].depth >= schema_.scopes[scope].depth ? sc : scope;
          int shallow = deep == sc ? scope : sc;
          int p = deep;
          while (p != 0 && p != shallow) p = schema_.scopes[p].parent;
          if (p != shallow) unsupported("expression over two unrelated iteration scopes", term->line);
          scope = deep;
        }
      } else {
        unsupported("internal: closure over a mixed value", term->line);
      }
      c->caps.emplace_back(v, a);
    }
    c->scope = scope;
    c->uses_data = touches_data(term);
    for (auto& cp : c->caps) c->uses_data = c->uses_data || (cp.second.k == CapArg::Col && cp.second.col->uses_data);
    std::string body;
    subst_print(*term, sub, body);
    // helper rules are identified by their TEXT (transitively), not by the template they live in: the same
    // `input_containers` partial set in two templates is one scope / one set of columns
    c->key = (refs_module(term) ? "r" + rules_signature(term) + ":" : std::string()) + body;
    return c;
  }

  // ---- product mode (second attempt of lower_violation): a collection iterated inside another, unrelated iteration becomes a
  // scope NESTED under the enclosing one (its generator is evaluated once per enclosing row), so that the two loop variables
  // lie on one scope chain and may be tested together -- `m := c.volumeMounts[_]; vol := spec.volumes[_]; vol.name == m.name`.
  // Rows are the cross product, as in the reference's nested iteration.
  struct IterGuard {
    std::vector<int>& st;
    IterGuard(std::vector<int>& s, int scope) : st(s) { st.push_back(scope); }
    ~IterGuard() { st.pop_back(); }
  };
  std::vector<int> iter_stack_;   // scopes whose EXISTS body is being lowered, outermost first
  int scope_of_collection(const CP& gen) {
    if (product_mode && !iter_stack_.empty()) {
      const int cur = iter_stack_.back();
      bool nested_in_cur = false;
      for (int p = gen->scope; p != 0; p = schema_.scopes[p].parent)
        if (p == cur) nested_in_cur = true;
      if (!nested_in_cur) {
        auto c = std::make_shared<Closure>(*gen);
        c->scope = cur;
        c->key = "@" + std::to_string(cur) + ":" + gen->key;
        return schema_.scope_for(c);
      }
    }
    return schema_.scope_for(gen);
  }

  CP leaf(int scope, bool is_key) {
    auto c = std::make_shared<Closure>();
    c->leaf = is_key ? Closure::Key : Closure::Elem;
    c->scope = scope;
    c->key = (is_key ? "$K" : "$E") + std::to_string(scope) + "{" + schema_.scopes[scope].gen->key + "}";
    return c;
  }

  TP synth_ref(const TP& head, std::vector<TP> path, int line) {
    auto t = std::make_shared<Term>();
    t->k = TK::Ref;
    t->head = head;
    t->args = std::move(path);
    t->line = line;
    synth_.push_back(t);
    return t;
  }
  TP synth_var(int vid, const std::string& name) {
    auto t = std::make_shared<Term>();
    t->k = TK::Var;
    t->vid = vid;
    t->name = name;
    synth_.push_back(t);
    return t;
  }
  TP synth_scalar(const VP& v) {
    auto t = std::make_shared<Term>();
    t->k = TK::Scalar;
    t->val = v;
    synth_.push_back(t);
    return t;
  }
  TP synth_call(const std::string& name, std::vector<TP> args, int line) {
    auto t = std::make_shared<Term>();
    t->k = TK::Call;
    t->name = name;
    t->args = std::move(args);
    t->line = line;
    synth_.push_back(t);
    return t;
  }

  // closure for  <col>[key]  /  f(<col>...)
  CP make_dot(const CP& base, const VP& key) {
    LEnv e;
    e.bind(vid_cur_, SymVal::column(base));
    return make_closure(synth_ref(synth_var(vid_cur_, "$cur"), {synth_scalar(key)}, 0), e);
  }
  CP make_call1(const std::string& fn, const CP& a) {
    LEnv e;
    e.bind(vid_cur_, SymVal::column(a));
    return make_closure(synth_call(fn, {synth_var(vid_cur_, "$cur")}, 0), e);
  }
  CP make_call2(const std::string& fn, const CP& a, const CP& b) {
    LEnv e;
    e.bind(vid_cur_, SymVal::column(a));
    e.bind(vid_key_, SymVal::column(b));
    return make_closure(synth_call(fn, {synth_var(vid_cur_, "$cur"), synth_var(vid_key_, "$key")}, 0), e);
  }

  // ------------------------------------------------------------------ atoms
  FP a_truthy(const CP& c) { return f_atom(GK_OP_TRUTHY, schema_.col_for(c, GK_ENC_VT)); }
  FP a_defined(const CP& c) { return f_atom(GK_OP_DEFINED, schema_.col_for(c, GK_ENC_VT)); }
  FP a_eq(const CP& c, const VP& v) { return f_atom(GK_OP_SID_EQ, schema_.col_for(c, GK_ENC_VT | GK_ENC_SID), v); }
  FP a_in(const CP& c, const VP& set) {
    if (set->items.empty()) return f_false();
    return f_atom(GK_OP_SID_IN, schema_.col_for(c, GK_ENC_VT | GK_ENC_SID), set);
  }
  // const c is a member of the collection-valued column S
  // existential over the elements of a symbolic collection (a collection-valued column or a SetOf)
  FP for_each_elem(const SymVal& S, int line, const std::function<FP(const SymVal& key, const SymVal& elem)>& body) {
    if (S.k == SymVal::Col) {
      int s = scope_of_collection(S.col);
      IterGuard g(iter_stack_, s);
      return f_exists(s, body(SymVal::column(leaf(s, true)), SymVal::column(leaf(s, false))));
    }
    if (S.k == SymVal::SetOf)
      return fill_tree(S.f, [&](uint32_t j) {
        const SymVal& h = S.items[j].second;
        FP d = defined_cond(h);
        if (d->k == Formula::False) return d;
        return f_and(d, body(h, h));
      });
    unsupported("iteration over this symbolic value", line);
  }
  FP fill_tree(const FP& f, const std::function<FP(uint32_t)>& fn) {
    switch (f->k) {
      case Formula::Atom: return f->op == -1 ? fn(f->imm) : f;
      case Formula::And: {
        FP o = f_true();
        for (auto& c : f->kids) o = f_and(o, fill_tree(c, fn));
        return o;
      }
      case Formula::Or: {
        FP o = f_false();
        for (auto& c : f->kids) o = f_or(o, fill_tree(c, fn));
        return o;
      }
      case Formula::Not: return f_not(fill_tree(f->kids[0], fn));
      case Formula::Exists: {
        IterGuard g(iter_stack_, f->scope);   // (the holes are filled inside the iteration: its rows are open there)
        return f->two ? f_exists2(f->scope, fill_tree(f->kids[0], fn)) : f_exists(f->scope, fill_tree(f->kids[0], fn));
      }
      default: return f;
    }
  }
  FP member_cond(const VP& c, const SymVal& S, int line) {
    return for_each_elem(S, line, [&](const SymVal&, const SymVal& e) { return eq_cond(e, SymVal::conc(c), line); });
  }
  FP in_const_cond(const SymVal& e, const VP& set, int line) {
    if (e.k == SymVal::Conc) return set_find(set, e.v) ? f_true() : f_false();
    if (e.k == SymVal::Col) return a_in(e.col, set);
    unsupported("membership of a composite symbolic value", line);
  }
  FP a_numcmp(const CP& c, uint32_t cmp, const VP& k, int line) {
    if (k->t != VT::Num) {
      // cross-type ordering against a non-number constant: only the rank matters unless the column is the same type
      unsupported("ordered comparison against a non-numeric parameter", line);
    }
    // Numeric columns hold num_key(x) = 2*floor(x) + (x is fractional): against an INTEGER constant every comparison is exact
    // for every object number.  A fractional threshold c (floor f) is the key 2f+1: exact against integer values and against
    // fractions with another integer part (a fraction with the SAME integer part as c compares as equal to it -- documented limit).
    int64_t dummy;
    if (!num_fits_i64(k->n, &dummy)) {
      const bool ordered = cmp == GK_CMP_LT || cmp == GK_CMP_LE || cmp == GK_CMP_GT || cmp == GK_CMP_GE;
      if (ordered && !k->n.is_int && std::isfinite(k->n.d) && std::fabs(k->n.d) < 2.0e18) {
        const uint32_t c2 = (cmp == GK_CMP_GT || cmp == GK_CMP_GE) ? (uint32_t)GK_CMP_GT : (uint32_t)GK_CMP_LT;
        return f_atom(GK_OP_NUM_CMP, schema_.col_for(c, GK_ENC_VT | GK_ENC_NUM), k, c2);
      }
      unsupported("ordered comparison against a parameter outside int64", line);
    }
    if (dummy > GK_NUM_KEY_CONST_LIMIT || dummy < -GK_NUM_KEY_CONST_LIMIT) unsupported("comparison against a parameter beyond 2^61", line);
    return f_atom(GK_OP_NUM_CMP, schema_.col_for(c, GK_ENC_VT | GK_ENC_NUM), k, cmp);
  }
  FP a_strop(int op, const CP& c, const VP& k) {
    // prefix tests run on the fixed-width HEAD record; the row's full bytes are only materialised when some prefix is longer
    // than the 31 bytes the record holds
    auto prefix_enc = [](const VP& list) {
      uint32_t enc = GK_ENC_VT | GK_ENC_HEAD;
      for (auto& x : list->items)
        if (x->t == VT::Str && x->s.size() > GK_HEAD_BYTES) enc |= GK_ENC_BYTES;
      return enc;
    };
    if (op == GK_OP_PREFIX) return f_atom(GK_OP_ANYPREFIX, schema_.col_for(c, prefix_enc(v_arr({k}))), v_arr({k}));
    if (op == GK_OP_ANYPREFIX) return f_atom(op, schema_.col_for(c, prefix_enc(k)), k);
    return f_atom(op, schema_.col_for(c, GK_ENC_VT | GK_ENC_BYTES), k);
  }

  FP defined_cond(const SymVal& v) {
    switch (v.k) {
      case SymVal::Conc: return f_true();
      case SymVal::Col: return v.col->leaf != Closure::None ? f_true() : a_defined(v.col);
      case SymVal::Bool: return v.d ? v.d : f_true();
      case SymVal::Opaque: return v.f ? v.f : f_true();
      case SymVal::Count: {
        const SymVal& x = v.items[0].second;   // count() of a column is undefined unless it holds a collection or a string
        return x.k == SymVal::Col ? a_defined(make_call1("count", x.col)) : f_true();
      }
      case SymVal::Arr: {
        if (v.compr) return f_true();
        FP f = f_true();
        for (auto& it : v.items) f = f_and(f, f_or(f_not(it.first), defined_cond(it.second)));
        return f;
      }
      case SymVal::ObjLit: {
        FP f = f_true();
        for (auto& it : v.fields) f = f_and(f, defined_cond(it.second));
        return f;
      }
      default: return f_true();
    }
  }

  // is element `it` of array `arr` there?  (a comprehension drops heads that are undefined; a literal array is all or nothing)
  FP present(const SymVal& arr, const std::pair<FP, SymVal>& it) {
    if (!arr.compr || it.second.k != SymVal::Bool || !it.second.d) return it.first;
    return f_and(it.first, it.second.d);
  }
  FP is_true_cond(const SymVal& v, int line) {
    if (v.k == SymVal::Bool) return v.f;
    if (v.k == SymVal::Conc) return v.v->t == VT::True ? f_true() : f_false();
    if (v.k == SymVal::Col) return f_atom(GK_OP_VTMASK, schema_.col_for(v.col, GK_ENC_VT), nullptr, 1u << GK_VT_TRUE);
    unsupported("any() / all() over non-boolean symbolic elements", line);
  }
  FP a_is_string(const CP& c) { return f_atom(GK_OP_VTMASK, schema_.col_for(c, GK_ENC_VT), nullptr, 1u << GK_VT_STR); }

  FP truthy_cond(const SymVal& v) {
    switch (v.k) {
      case SymVal::Conc: return v.v->t == VT::False ? f_false() : f_true();
      case SymVal::Col: return a_truthy(v.col);
      case SymVal::Bool: return v.f;
      case SymVal::Opaque: return v.f ? v.f : f_true();
      default: return defined_cond(v);
    }
  }

  // ------------------------------------------------------------------ concrete evaluation of param-only terms
  struct Alt {
    VP val;
    std::vector<std::pair<int, VP>> binds;
  };
  std::vector<Alt> concrete_solve(const TP& term, const LEnv& env) {
    Env ce;
    for (auto& b : env.b)
      if (b.second.k == SymVal::Conc) ce.bind(b.first, b.second.v);
    size_t base = ce.mark();
    std::vector<Alt> out;
    ev_.eval_term(term, ce, [&](const VP& v) {
      Alt a;
      a.val = v;
      for (size_t i = base; i < ce.b.size(); ++i) a.binds.push_back(ce.b[i]);
      out.push_back(std::move(a));
      if (out.size() > 4096) throw RegoError{"rego_unsupported: parameter iteration too large"};
      return false;
    });
    return out;
  }

  // ------------------------------------------------------------------ bodies
  FP lower_body(const std::vector<Stmt>& body, size_t i, LEnv& env, const BodyK& k) {
    if (i == body.size()) return k(env);
    const Stmt& st = body[i];
    auto rest = [&](LEnv& e) { return lower_body(body, i + 1, e, k); };
    switch (st.k) {
      case Stmt::Every: unsupported("internal: `every` reaches the lowering (the parser rewrites it)", st.line);
      case Stmt::Some: return rest(env);
      case Stmt::Not: {
        size_t mk = env.mark();
        FP inner = lower_expr(st.a, env, [](LEnv&) { return f_true(); });
        env.undo(mk);
        FP n = f_not(inner);
        if (n->k == Formula::False) return n;
        return f_and(n, rest(env));
      }
      case Stmt::Expr: return lower_expr(st.a, env, rest);
      case Stmt::Assign:
      case Stmt::Unify: return lower_unify(st.a, st.b, env, rest, st.line);
      case Stmt::SomeIn:
        return sym_term(st.c, env, [&](const SymVal& coll) { return iterate(coll, st.a, st.b, env, rest, st.line); });
    }
    return f_false();
  }

  FP lower_expr(const TP& t, LEnv& env, const BodyK& k) {
    Deps d = deps(t, env, false);
    if (pure_conc(d)) {
      FP out = f_false();
      for (auto& alt : concrete_solve(t, env)) {
        if (alt.val->t == VT::False) continue;
        size_t mk = env.mark();
        for (auto& b : alt.binds) env.bind(b.first, SymVal::conc(b.second, d.param));
        out = f_or(out, k(env));
        env.undo(mk);
      }
      return out;
    }
    return sym_term(t, env, [&](const SymVal& v) {
      FP c = truthy_cond(v);
      if (c->k == Formula::False) return c;
      return f_and(c, k(env));
    });
  }

  bool has_unbound(const TP& t, const LEnv& env) const {
    switch (t->k) {
      case TK::Var: return unbound(*t, env);
      case TK::Array:
      case TK::Set:
        for (auto& a : t->args)
          if (has_unbound(a, env)) return true;
        return false;
      case TK::Object:
        for (auto& kv : t->kvs)
          if (has_unbound(kv.first, env) || has_unbound(kv.second, env)) return true;
        return false;
      default: return false;
    }
  }

  FP lower_unify(const TP& a, const TP& b, LEnv& env, const BodyK& k, int line) {
    bool ua = has_unbound(a, env), ub = has_unbound(b, env);
    if (ua && !ub) return sym_term(b, env, [&](const SymVal& v) { return unify_pattern(a, v, env, k, line); });
    if (ub && !ua) return sym_term(a, env, [&](const SymVal& v) { return unify_pattern(b, v, env, k, line); });
    if (ua && ub) unsupported("unification of two non-ground terms", line);
    return lower_expr(synth_call("equal", {a, b}, line), env, k);
  }

  FP eq_cond(const SymVal& a, const SymVal& b, int line) {
    if (a.k == SymVal::Conc && b.k == SymVal::Conc) return v_eq(a.v, b.v) ? f_true() : f_false();
    if (a.k == SymVal::Col && b.k == SymVal::Conc) return a_eq(a.col, b.v);
    if (a.k == SymVal::Conc && b.k == SymVal::Col) return a_eq(b.col, a.v);
    if (a.k == SymVal::Col && b.k == SymVal::Col) return a_truthy(make_call2("equal", a.col, b.col));
    if (a.k == SymVal::Bool && b.k == SymVal::Conc) {
      if (b.v->t == VT::True) return a.f;
      if (b.v->t == VT::False) return f_and(defined_cond(a), f_not(a.f));
      return f_false();   // a boolean never equals a non-boolean
    }
    if (b.k == SymVal::Bool && a.k == SymVal::Conc) return eq_cond(b, a, line);
    if (a.k == SymVal::Count || b.k == SymVal::Count) return count_cmp(GK_CMP_EQ, a, b, line);
    if (a.k == SymVal::Opaque && a.col && b.k == SymVal::Conc) return a_eq(a.col, b.v);   // a formatted string against a constant
    if (b.k == SymVal::Opaque && b.col && a.k == SymVal::Conc) return a_eq(b.col, a.v);
    unsupported("equality between composite symbolic values", line);
  }

  FP unify_pattern(const TP& pat, const SymVal& v, LEnv& env, const BodyK& k, int line) {
    if (pat->k == TK::Var && unbound(*pat, env)) {
      FP c = defined_cond(v);
      if (c->k == Formula::False) return c;
      size_t mk = env.mark();
      env.bind(pat->vid, v);
      FP r = f_and(c, k(env));
      env.undo(mk);
      return r;
    }
    if (!has_unbound(pat, env)) {
      return sym_term(pat, env, [&](const SymVal& pv) {
        FP c = eq_cond(pv, v, line);
        if (c->k == Formula::False) return c;
        return f_and(c, k(env));
      });
    }
    if (v.k == SymVal::Conc) {
      // concrete unification of a composite pattern
      Env ce;
      for (auto& b : env.b)
        if (b.second.k == SymVal::Conc) ce.bind(b.first, b.second.v);
      size_t base = ce.mark();
      std::vector<std::vector<std::pair<int, VP>>> alts;
      ev_.unify_val(pat, v.v, ce, [&]() {
        alts.emplace_back(ce.b.begin() + base, ce.b.end());
        return false;
      });
      FP out = f_false();
      for (auto& al : alts) {
        size_t mk = env.mark();
        for (auto& b : al) env.bind(b.first, SymVal::conc(b.second, v.tainted));
        out = f_or(out, k(env));
        env.undo(mk);
      }
      return out;
    }
    if (pat->k == TK::Object && (v.k == SymVal::ObjLit || v.k == SymVal::Col)) {
      std::function<FP(size_t)> rec = [&](size_t i) -> FP {
        if (i == pat->kvs.size()) return k(env);
        const TP& kt = pat->kvs[i].first;
        if (kt->k != TK::Scalar) unsupported("non-constant key in object pattern", line);
        SymVal field;
        if (v.k == SymVal::ObjLit) {
          bool found = false;
          for (auto& f : v.fields)
            if (v_eq(f.first, kt->val)) {
              field = f.second;
              found = true;
            }
          if (!found) return f_false();
        } else {
          field = SymVal::column(make_dot(v.col, kt->val));
        }
        return unify_pattern(pat->kvs[i].second, field, env, [&](LEnv&) { return rec(i + 1); }, line);
      };
      if (v.k == SymVal::ObjLit && v.fields.size() != pat->kvs.size()) return f_false();
      return rec(0);
    }
    unsupported("pattern unification against a symbolic value", line);
  }

  // iterate `coll`, binding key pattern kp (may be null) and value pattern vp
  FP iterate(const SymVal& coll, const TP& kp, const TP& vp, LEnv& env, const BodyK& k, int line) {
    auto each = [&](const SymVal& key, const SymVal& val) -> FP {
      if (kp) return unify_pattern(kp, key, env, [&](LEnv&) { return unify_pattern(vp, val, env, k, line); }, line);
      return unify_pattern(vp, val, env, k, line);
    };
    switch (coll.k) {
      case SymVal::Conc: {
        FP out = f_false();
        const VP& c = coll.v;
        if (c->t == VT::Arr)
          for (size_t j = 0; j < c->items.size(); ++j) out = f_or(out, each(SymVal::conc(v_int((long long)j), coll.tainted), SymVal::conc(c->items[j], coll.tainted)));
        else if (c->t == VT::Set)
          for (auto& x : c->items) out = f_or(out, each(SymVal::conc(x, coll.tainted), SymVal::conc(x, coll.tainted)));
        else if (c->t == VT::Obj)
          for (auto& e : c->kv) out = f_or(out, each(SymVal::conc(e.first, coll.tainted), SymVal::conc(e.second, coll.tainted)));
        return out;
      }
      case SymVal::Col: {
        int s = scope_of_collection(coll.col);
        IterGuard g(iter_stack_, s);
        return f_exists(s, each(SymVal::column(leaf(s, true)), SymVal::column(leaf(s, false))));
      }
      case SymVal::Arr: {
        FP out = f_false();
        for (size_t j = 0; j < coll.items.size(); ++j)
          out = f_or(out, f_and(present(coll, coll.items[j]), each(SymVal::conc(v_int((long long)j)), coll.items[j].second)));
        return out;
      }
      case SymVal::DiffCS: {
        FP out = f_false();
        for (auto& x : coll.v->items) out = f_or(out, f_and(f_not(member_cond(x, *coll.sym, line)), each(SymVal::conc(x, true), SymVal::conc(x, true))));
        return out;
      }
      case SymVal::DiffSC:
        return for_each_elem(*coll.sym, line, [&](const SymVal&, const SymVal& e) { return f_and(f_not(in_const_cond(e, coll.v, line)), each(e, e)); });
      case SymVal::SetOf:
        return for_each_elem(coll, line, [&](const SymVal& kk, const SymVal& e) { return each(kk, e); });
      default: unsupported("iteration over this symbolic value", line);
    }
  }

  // ------------------------------------------------------------------ terms
  FP sym_term(const TP& t, LEnv& env, const SymK& k) {
    Deps d = deps(t, env, false);
    if (pure_conc(d)) {
      FP out = f_false();
      for (auto& alt : concrete_solve(t, env)) {
        size_t mk = env.mark();
        for (auto& b : alt.binds) env.bind(b.first, SymVal::conc(b.second, d.param));
        out = f_or(out, k(SymVal::conc(alt.val, d.param)));
        env.undo(mk);
      }
      return out;
    }
    // data.inventory (referential constraints): anything that reads the synced cache is evaluated by the host flattener, with the
    // constraint's parameters captured as constants -- joins over the inventory have no symbolic form here
    if (d.data && !d.iter && !schema_.device_only && t->k != TK::Var && !(t->k == TK::Call && t->name == "sprintf") && closable(t, env))
      return k(SymVal::column(make_closure(t, env)));
    if (pure_obj(d) && !(t->k == TK::Call && t->name == "sprintf") && t->k != TK::Array && t->k != TK::Object && t->k != TK::Set) {
      if (t->k == TK::Var) {
        if (const SymVal* s = env.find(t->vid)) {
          SymVal copy = *s;
          return k(copy);
        }
      }
      // device ingest: keep the closure only when the ingest kernels can compute it (a path, a count, a pure function of
      // leaf values); helper rules, comprehensions and impure functions are inlined below like their parameter-mixing kin
      if (!schema_.device_only) return k(SymVal::column(make_closure(t, env)));
      // (a comparison / string test against a constant is better an atom on the operand's column than a lookup column)
      static const std::set<std::string> kAtomic = {"equal", "neq", "lt", "lte", "gt", "gte", "startswith", "endswith", "contains",
                                                    "strings.any_prefix_match", "strings.any_suffix_match", "internal.member_2", "count"};
      if (!(t->k == TK::Call && !m_.is_rule(t->name) && kAtomic.count(t->name))) {
        CP cl = make_closure(t, env);
        if (closure_xinfo(*cl).k != XK::Host) return k(SymVal::column(cl));
      }
    }
    switch (t->k) {
      case TK::Var: {
        if (const SymVal* s = env.find(t->vid)) {
          SymVal copy = *s;
          return k(copy);
        }
        if (m_.is_rule(t->name)) return inline_rule_value(t, env, k);
        if (t->vid == m_.vid_input) {
          // the whole input document: {"parameters": <constant>, "review": <the object side>} -- e.g. the argument of
          // object.get(input, "parameters", {}) (test/gator/verify/template.yaml:23)
          SymVal doc;
          doc.k = SymVal::ObjLit;
          doc.fields.emplace_back(v_str("parameters"), SymVal::conc(params_, true));
          LEnv none;
          doc.fields.emplace_back(v_str("review"), SymVal::column(make_closure(synth_ref(synth_var(m_.vid_input, "input"), {synth_scalar(v_str("review"))}, t->line), none)));
          return k(doc);
        }
        unsupported("unbound variable " + t->name, t->line);
      }
      case TK::Ref: return sym_ref(t, env, k);
      case TK::Call: return sym_call(t, env, k);
      case TK::Array:
      case TK::Set: {
        SymVal arr;
        arr.k = SymVal::Arr;
        std::function<FP(size_t)> rec = [&](size_t i) -> FP {
          if (i == t->args.size()) return k(arr);
          return sym_term(t->args[i], env, [&](const SymVal& v) {
            arr.items.emplace_back(f_true(), v);
            FP r = rec(i + 1);
            arr.items.pop_back();
            return r;
          });
        };
        return rec(0);
      }
      case TK::Object: {
        SymVal obj;
        obj.k = SymVal::ObjLit;
        std::function<FP(size_t)> rec = [&](size_t i) -> FP {
          if (i == t->kvs.size()) return k(obj);
          return sym_term(t->kvs[i].first, env, [&](const SymVal& kv) {
            if (kv.k != SymVal::Conc) unsupported("symbolic object key", t->line);
            return sym_term(t->kvs[i].second, env, [&](const SymVal& vv) {
              obj.fields.emplace_back(kv.v, vv);
              FP r = rec(i + 1);
              obj.fields.pop_back();
              return r;
            });
          });
        };
        return rec(0);
      }
      case TK::ArrCompr: return sym_arr_compr(t, env, k);
      case TK::SetCompr: return sym_set_compr(t, env, k);
      default: unsupported("set/object comprehension mixing parameters and object fields", t->line);
    }
  }

  // [head | body] whose body mixes parameters and object fields: concrete-length result, symbolic elements
  FP sym_arr_compr(const TP& t, LEnv& env, const SymK& k) {
    std::vector<SymVal> vals;
    size_t mk = env.mark();
    FP tree = lower_body(t->body, 0, env, [&](LEnv& e) {
      return sym_term(t->value, e, [&](const SymVal& v) {
        vals.push_back(v);
        auto h = std::make_shared<Formula>();
        h->k = Formula::Atom;
        h->op = -1;                       // hole marker
        h->imm = (uint32_t)vals.size() - 1;
        return FP(h);
      });
    });
    env.undo(mk);
    SymVal arr;
    arr.k = SymVal::Arr;
    arr.compr = true;
    try {
      for (size_t j = 0; j < vals.size(); ++j) {
        FP guard = fill_holes(tree, (uint32_t)j, t->line);
        arr.items.emplace_back(guard, vals[j]);
      }
    } catch (RegoError& e) {
      if (e.msg.find("comprehension over an object collection mixed with parameters") == std::string::npos) throw;
      SymVal h;
      h.k = SymVal::ArrHoles;
      h.f = tree;
      for (auto& v : vals) h.items.emplace_back(f_true(), v);
      return k(h);
    }
    return k(arr);
  }
  // {head | body} whose body mixes parameters and object fields: kept as a formula with one hole per way of
  // producing an element; membership / emptiness tests substitute the hole (see for_each_elem)
  FP sym_set_compr(const TP& t, LEnv& env, const SymK& k) {
    SymVal set;
    set.k = SymVal::SetOf;
    size_t mk = env.mark();
    set.f = lower_body(t->body, 0, env, [&](LEnv& e) {
      return sym_term(t->value, e, [&](const SymVal& v) {
        if (v.k != SymVal::Col && v.k != SymVal::Conc) unsupported("set comprehension over composite symbolic values", t->line);
        set.items.emplace_back(f_true(), v);
        auto h = std::make_shared<Formula>();
        h->k = Formula::Atom;
        h->op = -1;
        h->imm = (uint32_t)set.items.size() - 1;
        return FP(h);
      });
    });
    env.undo(mk);
    return k(set);
  }
  FP fill_holes(const FP& f, uint32_t which, int line) {
    switch (f->k) {
      case Formula::Atom:
        if (f->op == -1) return f->imm == which ? f_true() : f_false();
        return f;
      case Formula::And: {
        FP o = f_true();
        for (auto& c : f->kids) o = f_and(o, fill_holes(c, which, line));
        return o;
      }
      case Formula::Or: {
        FP o = f_false();
        for (auto& c : f->kids) o = f_or(o, fill_holes(c, which, line));
        return o;
      }
      case Formula::Not: return f_not(fill_holes(f->kids[0], which, line));
      case Formula::Exists: unsupported("comprehension over an object collection mixed with parameters", line);
      default: return f;
    }
  }

  // complete rule referenced by name whose definition mixes parameters and object fields
  FP inline_rule_value(const TP& t, LEnv& /*env*/, const SymK& k) {
    auto& defs = m_.rules.at(t->name);
    if (defs[0].kind != Rule::Complete) unsupported("partial rule `" + t->name + "` used as a value while mixing parameters and object fields", t->line);
    if (++depth_ > 24) unsupported("rule nesting too deep", t->line);
    FP out = f_false();
    for (auto& r : defs) {
      if (r.is_default || !r.els.empty()) unsupported("default/else rule mixing parameters and object fields", r.line);
      LEnv fe;
      out = f_or(out, lower_body(r.body, 0, fe, [&](LEnv& e) { return sym_term(r.value, e, k); }));
    }
    --depth_;
    return out;
  }

  FP sym_ref(const TP& t, LEnv& env, const SymK& k) {
    // partial set/object rule that mixes parameters and object fields: inline its definitions
    if (t->head->k == TK::Var && !env.find(t->head->vid) && m_.is_rule(t->head->name)) {
      auto& defs = m_.rules.at(t->head->name);
      Deps rd = rule_deps(t->head->name);
      if ((defs[0].kind == Rule::PSet || defs[0].kind == Rule::PObj) && !((pure_obj(rd) && !schema_.device_only) || pure_conc(rd)))
        return inline_partial(t, env, k);
    }
    // longest prefix that is purely parameters or purely object
    for (size_t j = t->args.size(); j-- > 0;) {
      TP prefix = j == 0 ? t->head : synth_ref(t->head, std::vector<TP>(t->args.begin(), t->args.begin() + j), t->line);
      Deps d = deps(prefix, env, false);
      if (d.iter) continue;
      if (pure_conc(d) || pure_obj(d) || j == 0) {
        return sym_term(prefix, env, [&](const SymVal& base) { return walk_sym(base, t->args, j, env, k, t->line); });
      }
    }
    unsupported("reference", t->line);
  }

  FP inline_partial(const TP& t, LEnv& env, const SymK& k) {
    auto& defs = m_.rules.at(t->head->name);
    if (t->args.empty()) unsupported("partial rule used as a whole value", t->line);
    if (++depth_ > 24) unsupported("rule nesting too deep", t->line);
    const TP& p0 = t->args[0];
    FP out = f_false();
    for (auto& r : defs) {
      LEnv fe;
      // pre-bind head variables from constant parts of the call-site pattern (a filter on the head var)
      if (p0->k == TK::Object && r.key->k == TK::Object) {
        for (auto& pk : p0->kvs)
          for (auto& rk : r.key->kvs)
            if (pk.first->k == TK::Scalar && rk.first->k == TK::Scalar && v_eq(pk.first->val, rk.first->val) &&
                pk.second->k == TK::Scalar && rk.second->k == TK::Var && unbound(*rk.second, fe))
              fe.bind(rk.second->vid, SymVal::conc(pk.second->val));
      }
      FP f = lower_body(r.body, 0, fe, [&](LEnv& e) {
        return sym_term(r.key, e, [&](const SymVal& kv) {
          auto cont = [&](LEnv&) {
            if (defs[0].kind == Rule::PObj) return sym_term(r.value, e, [&](const SymVal& vv) { return walk_sym(vv, t->args, 1, env, k, t->line); });
            return walk_sym(kv, t->args, 1, env, k, t->line);
          };
          return unify_pattern(p0, kv, env, cont, t->line);
        });
      });
      out = f_or(out, f);
    }
    --depth_;
    return out;
  }

  FP walk_sym(const SymVal& cur, const std::vector<TP>& path, size_t i, LEnv& env, const SymK& k, int line) {
    if (i == path.size()) return k(cur);
    const TP& p = path[i];
    auto next = [&](const SymVal& v) { return walk_sym(v, path, i + 1, env, k, line); };
    if (has_unbound(p, env)) {
      // iteration (plain variable / wildcard) or pattern key
      TP keypat = p;
      return iterate_keyed(cur, keypat, env, next, line);
    }
    return sym_term(p, env, [&](const SymVal& kv) -> FP {
      switch (cur.k) {
        case SymVal::Conc: {
          if (kv.k == SymVal::Conc) {
            VP got;
            const VP& c = cur.v;
            if (c->t == VT::Obj) got = obj_get(c, kv.v);
            else if (c->t == VT::Arr) {
              int64_t ix;
              if (kv.v->t == VT::Num && num_fits_i64(kv.v->n, &ix) && ix >= 0 && (size_t)ix < c->items.size()) got = c->items[ix];
            } else if (c->t == VT::Set) got = set_find(c, kv.v);
            if (!got) return f_false();
            return next(SymVal::conc(got, cur.tainted || kv.tainted));
          }
          if (kv.k == SymVal::Col && cur.v->t == VT::Set) {
            FP c = a_in(kv.col, cur.v);
            if (c->k == Formula::False) return c;
            return f_and(c, next(kv));
          }
          if (kv.k == SymVal::Col && cur.v->t == VT::Obj) {
            // obj[col]: value depends on which key matched -> one alternative per key
            FP out = f_false();
            for (auto& e : cur.v->kv) out = f_or(out, f_and(a_eq(kv.col, e.first), next(SymVal::conc(e.second, cur.tainted))));
            return out;
          }
          unsupported("index of a constant by a symbolic value", line);
        }
        case SymVal::Col: {
          if (kv.k == SymVal::Conc) return next(SymVal::column(make_dot(cur.col, kv.v)));
          if (kv.k == SymVal::Col) {
            LEnv e;
            e.bind(vid_cur_, cur);
            e.bind(vid_key_, kv);
            return next(SymVal::column(make_closure(synth_ref(synth_var(vid_cur_, "$cur"), {synth_var(vid_key_, "$key")}, line), e)));
          }
          unsupported("index of an object field by a mixed value", line);
        }
        case SymVal::ObjLit: {
          if (kv.k != SymVal::Conc) unsupported("symbolic key into object literal", line);
          for (auto& f : cur.fields)
            if (v_eq(f.first, kv.v)) return next(f.second);
          return f_false();
        }
        case SymVal::Arr: {
          int64_t ix;
          if (kv.k != SymVal::Conc || kv.v->t != VT::Num || !num_fits_i64(kv.v->n, &ix)) unsupported("symbolic index", line);
          if (ix < 0 || (size_t)ix >= cur.items.size()) return f_false();
          // positions shift when guards are false: only exact when every earlier guard is constant true
          for (int64_t j = 0; j <= ix; ++j)
            if (cur.items[j].first->k != Formula::True) unsupported("index into a conditionally-built array", line);
          return next(cur.items[ix].second);
        }
        case SymVal::DiffCS: {
          if (kv.k != SymVal::Conc) unsupported("symbolic membership in a set difference", line);
          if (!set_find(cur.v, kv.v)) return f_false();
          return f_and(f_not(member_cond(kv.v, *cur.sym, line)), next(kv));
        }
        default: unsupported("reference into this symbolic value", line);
      }
    });
  }

  // x[p] where p contains unbound variables: iterate x and unify p with each key (sets: the element)
  FP iterate_keyed(const SymVal& cur, const TP& keypat, LEnv& env, const SymK& next, int line) {
    auto each = [&](const SymVal& key, const SymVal& val) -> FP {
      return unify_pattern(keypat, key, env, [&](LEnv&) { return next(val); }, line);
    };
    switch (cur.k) {
      case SymVal::Conc: {
        FP out = f_false();
        const VP& c = cur.v;
        if (c->t == VT::Arr)
          for (size_t j = 0; j < c->items.size(); ++j) out = f_or(out, each(SymVal::conc(v_int((long long)j), cur.tainted), SymVal::conc(c->items[j], cur.tainted)));
        else if (c->t == VT::Set)
          for (auto& x : c->items) out = f_or(out, each(SymVal::conc(x, cur.tainted), SymVal::conc(x, cur.tainted)));
        else if (c->t == VT::Obj)
          for (auto& e : c->kv) out = f_or(out, each(SymVal::conc(e.first, cur.tainted), SymVal::conc(e.second, cur.tainted)));
        return out;
      }
      case SymVal::Col: {
        int s = scope_of_collection(cur.col);
        IterGuard g(iter_stack_, s);
        return f_exists(s, each(SymVal::column(leaf(s, true)), SymVal::column(leaf(s, false))));
      }
      case SymVal::Arr: {
        FP out = f_false();
        for (size_t j = 0; j < cur.items.size(); ++j) {
          if (cur.items[j].first->k != Formula::True && keypat->k == TK::Var && keypat->name[0] != '$')
            unsupported("index variable over a conditionally-built array", line);
          out = f_or(out, f_and(present(cur, cur.items[j]), each(SymVal::conc(v_int((long long)j)), cur.items[j].second)));
        }
        return out;
      }
      case SymVal::DiffCS: {
        FP out = f_false();
        for (auto& x : cur.v->items) out = f_or(out, f_and(f_not(member_cond(x, *cur.sym, line)), each(SymVal::conc(x, true), SymVal::conc(x, true))));
        return out;
      }
      case SymVal::DiffSC:
        return for_each_elem(*cur.sym, line, [&](const SymVal&, const SymVal& e) { return f_and(f_not(in_const_cond(e, cur.v, line)), each(e, e)); });
      case SymVal::SetOf:
        return for_each_elem(cur, line, [&](const SymVal& kk, const SymVal& e) { return each(kk, e); });
      default: unsupported("iteration over this symbolic value", line);
    }
  }

  // ------------------------------------------------------------------ calls
  FP sym_call(const TP& t, LEnv& env, const SymK& k) {
    auto rit = m_.rules.find(t->name);
    bool user = rit != m_.rules.end();
    if (user && rit->second[0].kind != Rule::Func) throw RegoError{"rego_type_error: " + t->name + " is not a function"};
    size_t nformal = user ? rit->second[0].args.size() : t->args.size();
    if (user && t->args.size() != nformal) unsupported("function call with output argument", t->line);
    std::vector<SymVal> args;
    // a sprintf over object fields only is normally just a message (never a column: it would be computed for every object);
    // it carries its closure along so that a COMPARISON with a constant can still become a column atom
    CP text_closure;
    if (!user && t->name == "sprintf" && pure_obj(deps(t, env, false))) {
      try {
        text_closure = make_closure(t, env);
      } catch (RegoError&) {
      }
    }
    SymK k2 = [&](const SymVal& v) {
      if (!text_closure || v.k != SymVal::Opaque) return k(v);
      SymVal w = v;
      w.col = text_closure;
      return k(w);
    };
    std::function<FP(size_t)> rec = [&](size_t i) -> FP {
      if (i == t->args.size()) return user ? inline_function(t, args, k) : builtin_sym(t, args, text_closure ? k2 : k);
      return sym_term(t->args[i], env, [&](const SymVal& v) {
        args.push_back(v);
        FP r = rec(i + 1);
        args.pop_back();
        return r;
      });
    };
    return rec(0);
  }

  FP inline_function(const TP& t, const std::vector<SymVal>& args, const SymK& k) {
    if (++depth_ > 24) unsupported("function nesting too deep (recursion?)", t->line);
    FP out = f_false();
    for (auto& r : m_.rules.at(t->name)) {
      if (r.args.size() != args.size()) continue;
      if (!r.els.empty()) unsupported("`else` in a function that mixes parameters and object fields", r.line);
      LEnv fe;
      std::function<FP(size_t)> bind = [&](size_t i) -> FP {
        if (i == args.size()) return lower_body(r.body, 0, fe, [&](LEnv& e) { return sym_term(r.value, e, k); });
        return unify_pattern(r.args[i], args[i], fe, [&](LEnv&) { return bind(i + 1); }, r.line);
      };
      out = f_or(out, bind(0));
      check_size(out, t->line);
    }
    --depth_;
    return out;
  }

  static uint32_t flip_cmp(uint32_t c) {
    switch (c) {
      case GK_CMP_LT: return GK_CMP_GT;
      case GK_CMP_LE: return GK_CMP_GE;
      case GK_CMP_GT: return GK_CMP_LT;
      case GK_CMP_GE: return GK_CMP_LE;
      default: return c;
    }
  }

  // count(X) <cmp> n  (X symbolic collection, n constant) or flipped
  FP count_cmp(uint32_t cmp, const SymVal& a, const SymVal& b, int line) {
    if (a.k != SymVal::Count) {
      if (b.k != SymVal::Count) unsupported("count comparison", line);
      return count_cmp(flip_cmp(cmp), b, a, line);
    }
    if (b.k != SymVal::Conc || b.v->t != VT::Num) unsupported("count compared with a non-constant", line);
    int64_t n;
    if (!num_fits_i64(b.v->n, &n)) unsupported("count compared with a huge constant", line);
    const SymVal& x = a.items[0].second;
    // normalise to: at-least(k) / at-most(k) / exactly(k)
    std::vector<FP> bools;
    bool scoped = false;
    FP any_scoped;
    if (x.k == SymVal::DiffCS) {
      for (auto& c : x.v->items) bools.push_back(f_not(member_cond(c, *x.sym, line)));
    } else if (x.k == SymVal::Arr) {
      for (auto& it : x.items) bools.push_back(present(x, it));
    } else if (x.k == SymVal::DiffSC) {
      scoped = true;
      any_scoped = for_each_elem(*x.sym, line, [&](const SymVal&, const SymVal& e) { return f_not(in_const_cond(e, x.v, line)); });
    } else if (x.k == SymVal::SetOf) {
      scoped = true;
      any_scoped = for_each_elem(x, line, [&](const SymVal&, const SymVal&) { return f_true(); });
    } else if (x.k == SymVal::ArrHoles) {
      scoped = true;
      any_scoped = fill_tree(x.f, [&](uint32_t j) { return defined_cond(x.items[j].second); });
    } else if (x.k == SymVal::Col) {
      return a_numcmp(make_call1("count", x.col), cmp, b.v, line);
    } else {
      unsupported("count of this symbolic value", line);
    }
    auto any = [&]() -> FP {
      if (scoped) return any_scoped;
      FP o = f_false();
      for (auto& f : bools) o = f_or(o, f);
      return o;
    };
    auto all = [&]() -> FP {
      FP o = f_true();
      for (auto& f : bools) o = f_and(o, f);
      return o;
    };
    int64_t total = scoped ? -1 : (int64_t)bools.size();
    // count in [0, total]
    switch (cmp) {
      case GK_CMP_GT:
        if (n < 0) return f_true();
        if (n == 0) return any();
        if (!scoped && n >= total) return f_false();
        if (!scoped && n == total - 1) return all();
        break;
      case GK_CMP_GE:
        if (n <= 0) return f_true();
        if (n == 1) return any();
        if (!scoped && n > total) return f_false();
        if (!scoped && n == total) return all();
        break;
      case GK_CMP_LT:
        if (n <= 0) return f_false();
        if (n == 1) return f_not(any());
        if (!scoped && n > total) return f_true();
        if (!scoped && n == total) return f_not(all());
        break;
      case GK_CMP_LE:
        if (n < 0) return f_false();
        if (n == 0) return f_not(any());
        if (!scoped && n >= total) return f_true();
        if (!scoped && n == total - 1) return f_not(all());
        break;
      case GK_CMP_EQ:
        if (n < 0) return f_false();
        if (n == 0) return f_not(any());
        if (!scoped && n > total) return f_false();
        if (!scoped && n == total) return all();
        break;
      case GK_CMP_NE:
        if (n < 0) return f_true();
        if (n == 0) return any();
        if (!scoped && n > total) return f_true();
        if (!scoped && n == total) return f_not(all());
        break;
    }
    unsupported("count compared with a constant other than 0 / the full size", line);
  }

  FP builtin_sym(const TP& t, const std::vector<SymVal>& a, const SymK& k) {
    const std::string& n = t->name;
    const int line = t->line;
    auto is_conc = [](const SymVal& s) { return s.k == SymVal::Conc; };
    auto is_col = [](const SymVal& s) { return s.k == SymVal::Col; };
    // the value is defined only where every argument is (plus whatever type the builtin insists on: `extra`)
    auto ret_bool = [&](FP f, FP extra = nullptr) {
      FP d = extra ? extra : f_true();
      for (auto& x : a) d = f_and(d, defined_cond(x));
      return k(SymVal::boolean(std::move(f), d->k == Formula::True ? FP() : d));
    };
    auto undefined_bool = [&]() { return k(SymVal::boolean(f_false(), f_false())); };

    if (n == "print" || n == "trace") return k(SymVal::conc(v_bool(true)));
    if (n == "sprintf") {
      FP def = f_true();
      for (auto& x : a) def = f_and(def, defined_cond(x));
      if (def->k == Formula::False) return def;
      SymVal o = SymVal::opaque(def);
      for (auto& x : a) o.row_dep = o.row_dep || !object_level_val(x);   // (the text depends on the rows that are open here)
      return k(o);
    }
    if (n == "object.get" && a.size() == 3 && a[0].k == SymVal::ObjLit && is_conc(a[1])) {
      for (auto& f : a[0].fields)
        if (v_eq(f.first, a[1].v)) return k(f.second);
      return k(a[2]);
    }
    if (n == "equal" && a.size() == 2) return ret_bool(eq_cond(a[0], a[1], line));
    if (n == "neq" && a.size() == 2) {
      if (a[0].k == SymVal::Count || a[1].k == SymVal::Count) return ret_bool(count_cmp(GK_CMP_NE, a[0], a[1], line));
      FP eq = eq_cond(a[0], a[1], line);
      // `x != y` is undefined (not true) when an operand is undefined
      return ret_bool(f_and(f_and(defined_cond(a[0]), defined_cond(a[1])), f_not(eq)));
    }
    if ((n == "lt" || n == "lte" || n == "gt" || n == "gte") && a.size() == 2) {
      uint32_t cmp = n == "lt" ? GK_CMP_LT : n == "lte" ? GK_CMP_LE : n == "gt" ? GK_CMP_GT : GK_CMP_GE;
      if (a[0].k == SymVal::Count || a[1].k == SymVal::Count) return ret_bool(count_cmp(cmp, a[0], a[1], line));
      if (is_col(a[0]) && is_conc(a[1])) return ret_bool(a_numcmp(a[0].col, cmp, a[1].v, line));
      if (is_conc(a[0]) && is_col(a[1])) return ret_bool(a_numcmp(a[1].col, flip_cmp(cmp), a[0].v, line));
      if (is_col(a[0]) && is_col(a[1])) return ret_bool(a_truthy(make_call2(n, a[0].col, a[1].col)));
      unsupported("ordered comparison of composite symbolic values", line);
    }
    if (n == "count" && a.size() == 1) {
      SymVal c;
      c.k = SymVal::Count;
      c.items.emplace_back(f_true(), a[0]);
      if (a[0].k == SymVal::Opaque || a[0].k == SymVal::Bool || a[0].k == SymVal::ObjLit) unsupported("count of this value", line);
      return k(c);
    }
    if (n == "minus" && a.size() == 2) {
      auto is_symset = [](const SymVal& s) { return s.k == SymVal::Col || s.k == SymVal::SetOf; };
      if (is_conc(a[0]) && a[0].v->t == VT::Set && is_symset(a[1])) {
        SymVal d;
        d.k = SymVal::DiffCS;
        d.v = a[0].v;
        d.sym = std::make_shared<SymVal>(a[1]);
        return k(d);
      }
      if (is_symset(a[0]) && is_conc(a[1]) && a[1].v->t == VT::Set) {
        SymVal d;
        d.k = SymVal::DiffSC;
        d.v = a[1].v;
        d.sym = std::make_shared<SymVal>(a[0]);
        return k(d);
      }
      unsupported("arithmetic mixing parameters and object fields", line);
    }
    if ((n == "startswith" || n == "endswith" || n == "contains") && a.size() == 2) {
      int op = n == "startswith" ? GK_OP_PREFIX : n == "endswith" ? GK_OP_SUFFIX : GK_OP_CONTAINS;
      if (is_col(a[0]) && is_conc(a[1])) {
        if (a[1].v->t != VT::Str) return undefined_bool();   // type error => undefined
        return ret_bool(a_strop(op, a[0].col, a[1].v), a_is_string(a[0].col));
      }
      unsupported(n + " with a symbolic second operand", line);
    }
    if ((n == "strings.any_prefix_match" || n == "strings.any_suffix_match") && a.size() == 2) {
      if (is_col(a[0]) && is_conc(a[1])) {
        std::vector<VP> pats;
        const VP& b = a[1].v;
        if (b->t == VT::Str) pats.push_back(b);
        else if (b->t == VT::Arr || b->t == VT::Set) {
          for (auto& x : b->items) {
            if (x->t != VT::Str) return undefined_bool();
            pats.push_back(x);
          }
        } else {
          return undefined_bool();
        }
        if (pats.empty()) return ret_bool(f_false(), a_is_string(a[0].col));
        return ret_bool(a_strop(n == "strings.any_prefix_match" ? GK_OP_ANYPREFIX : GK_OP_ANYSUFFIX, a[0].col, v_arr(pats)), a_is_string(a[0].col));
      }
      unsupported(n + " with a symbolic pattern list", line);
    }
    if ((n == "any" || n == "all") && a.size() == 1 && a[0].k == SymVal::ArrHoles) {
      const SymVal& h = a[0];
      if (n == "any") return ret_bool(fill_tree(h.f, [&](uint32_t j) { return is_true_cond(h.items[j].second, line); }));
      return ret_bool(f_not(fill_tree(h.f, [&](uint32_t j) {
        return f_and(defined_cond(h.items[j].second), f_not(is_true_cond(h.items[j].second, line)));
      })));
    }
    if (n == "any" && a.size() == 1) {
      if (a[0].k != SymVal::Arr) unsupported("any() of this value", line);
      FP o = f_false();
      for (auto& it : a[0].items) o = f_or(o, f_and(it.first, is_true_cond(it.second, line)));   // (a true element is a defined one)
      return ret_bool(o);
    }
    if (n == "all" && a.size() == 1) {
      if (a[0].k != SymVal::Arr) unsupported("all() of this value", line);
      // false as soon as one element that is THERE is not `true`
      FP bad = f_false();
      for (auto& it : a[0].items) {
        FP there = a[0].compr ? f_and(it.first, defined_cond(it.second)) : it.first;
        bad = f_or(bad, f_and(there, f_not(is_true_cond(it.second, line))));
      }
      return ret_bool(f_not(bad));
    }
    if (n == "internal.member_2" && a.size() == 2) {
      if (is_col(a[0]) && is_conc(a[1])) {
        std::vector<VP> vals;
        if (a[1].v->t == VT::Obj)
          for (auto& e : a[1].v->kv) vals.push_back(e.second);
        else if (a[1].v->t == VT::Arr || a[1].v->t == VT::Set) vals = a[1].v->items;
        return ret_bool(f_and(a_defined(a[0].col), a_in(a[0].col, v_set(vals))));
      }
      if (is_conc(a[0]) && (is_col(a[1]) || a[1].k == SymVal::SetOf)) return ret_bool(member_cond(a[0].v, a[1], line));
      unsupported("`in` over this symbolic value", line);
    }
    if ((n == "re_match" || n == "regex.match") && a.size() == 2 && is_conc(a[0]) && is_col(a[1])) {
      // Regular expressions are not evaluated on the device: `re_match(<pattern from the parameters>, <object string>)`
      // becomes a boolean FEATURE COLUMN of its own -- the flattener runs the (cached, compiled) pattern once per row --
      // keyed by the pattern text, so constraints that share a pattern share the column.
      if (a[0].v->t != VT::Str) return undefined_bool();   // non-string pattern: undefined
      LEnv e;
      e.bind(vid_cur_, a[1]);
      CP c = make_closure(synth_call(n, {synth_scalar(a[0].v), synth_var(vid_cur_, "$cur")}, line), e);
      return ret_bool(f_atom(GK_OP_VTMASK, schema_.col_for(c, GK_ENC_VT), nullptr, 1u << GK_VT_TRUE), a_is_string(a[1].col));
    }
    if (n == "re_match" || n == "regex.match") unsupported("regular expression with a pattern taken from the object", line);
    unsupported("builtin " + n + " mixing parameters and object fields", line);
  }
};

void Lowerer::subst_print(const Term& t, const std::map<int, std::string>& sub, std::string& out) {
  // term_str with captured variables replaced by their canonical keys
  if (t.k == TK::Var) {
    auto it = sub.find(t.vid);
    if (it != sub.end()) out += it->second;
    else out += (t.name.size() > 1 && t.name[0] == '$' && t.name[1] == 'w') ? std::string("_") : t.name;
    return;
  }
  if (sub.empty()) {
    out += term_str(t);
    return;
  }
  // structural print (mirrors term_str) so nested vars are substituted
  switch (t.k) {
    case TK::Scalar: out += fmt_value(t.val, false); break;
    case TK::Ref:
      subst_print(*t.head, sub, out);
      for (auto& a : t.args) {
        out.push_back('[');
        subst_print(*a, sub, out);
        out.push_back(']');
      }
      break;
    case TK::Call:
      out += t.name + "(";
      for (size_t i = 0; i < t.args.size(); ++i) {
        if (i) out += ", ";
        subst_print(*t.args[i], sub, out);
      }
      out += ")";
      break;
    case TK::Array:
    case TK::Set:
      out += t.k == TK::Array ? "[" : "{";
      for (size_t i = 0; i < t.args.size(); ++i) {
        if (i) out += ", ";
        subst_print(*t.args[i], sub, out);
      }
      out += t.k == TK::Array ? "]" : "}";
      break;
    case TK::Object:
      out += "{";
      for (size_t i = 0; i < t.kvs.size(); ++i) {
        if (i) out += ", ";
        subst_print(*t.kvs[i].first, sub, out);
        out += ": ";
        subst_print(*t.kvs[i].second, sub, out);
      }
      out += "}";
      break;
    default: {
      // comprehensions: print head/body with substitution
      out += t.k == TK::ArrCompr ? "[" : "{";
      if (t.key) {
        subst_print(*t.key, sub, out);
        out += ": ";
      }
      subst_print(*t.value, sub, out);
      out += " | ";
      for (size_t i = 0; i < t.body.size(); ++i) {
        const Stmt& s = t.body[i];
        if (i) out += "; ";
        if (s.k == Stmt::Not) out += "not ";
        if (s.k == Stmt::Some) out += "some";
        if (s.a) subst_print(*s.a, sub, out);
        if (s.k == Stmt::Assign) out += " := ";
        if (s.k == Stmt::Unify) out += " = ";
        if (s.k == Stmt::SomeIn) out += " <- ";
        if (s.b) subst_print(*s.b, sub, out);
        if (s.c) {
          out += " in ";
          subst_print(*s.c, sub, out);
        }
      }
      out += t.k == TK::ArrCompr ? "]" : "}";
    }
  }
}

}  // namespace

FP lower_violation(const std::shared_ptr<const Module>& mod, const VP& parameters, Schema& schema, bool device_mode, bool* single_result, FP* amb) {
  schema.device_only = device_mode;
  const Schema before = schema;   // (a failed attempt must not leave its scopes and columns behind)
  if (single_result) *single_result = false;
  if (amb) *amb = f_true();
  try {
    Lowerer lw(mod, parameters, schema);
    FP f = lw.run();
    if (single_result) *single_result = lw.single_result();
    if (amb) *amb = lw.single_result() ? f_false() : lw.ambiguity();
    return f;
  } catch (RegoError& e) {
    if (e.msg.find("two unrelated iteration scopes") == std::string::npos) {
      schema = before;
      throw;
    }
  }
  schema = before;
  try {
    Lowerer lw(mod, parameters, schema);
    lw.product_mode = true;
    FP f = lw.run();
    if (single_result) *single_result = lw.single_result();
    if (amb) *amb = lw.single_result() ? f_false() : lw.ambiguity();
    return f;
  } catch (RegoError&) {
    schema = before;
    throw;
  }
}

// ====================================================================================== netlist construction
uint32_t NetBuilder::add_bytes(const std::string& s) {
  uint32_t off = (uint32_t)cbytes.size();
  cbytes.insert(cbytes.end(), s.begin(), s.end());
  return off;
}

namespace {

struct NNode {
  uint8_t kind = 0;        // GK_N_*
  int level = 0;           // scope of the rows this node has one bit for
  int a = -1, b = -1;      // input (BCAST / ACC)
  std::vector<std::pair<int, bool>> ins;   // GATE inputs: (node, negated)
  uint32_t flags = 0;      // gate flags / const value
  int scope = 0;           // BCAST / ACC: the child scope
  // atom
  int op = 0, col = -1;
  VP cval;
  uint32_t imm = 0;
  uint32_t match_id = 0;
  int err_of = -1;         // MATCH: id of the paired error node (a pseudo node that only owns a slot)
  int phase = 0, last_use = 0, slot = -1;
};

struct Ref {
  int node;
  bool neg;
};

struct Net {
  const Schema& schema;
  std::vector<NNode> nodes;
  std::map<std::string, int> memo;
  explicit Net(const Schema& s) : schema(s) {}

  int depth(int scope) const { return schema.scopes[scope].depth; }

  int intern_node(const std::string& key, NNode n) {
    auto it = memo.find(key);
    if (it != memo.end()) return it->second;
    n.phase = 0;
    if (n.a >= 0) n.phase = std::max(n.phase, nodes[n.a].phase + 1);
    if (n.b >= 0) n.phase = std::max(n.phase, nodes[n.b].phase + 1);
    for (auto& in : n.ins) n.phase = std::max(n.phase, nodes[in.first].phase + 1);
    nodes.push_back(std::move(n));
    int id = (int)nodes.size() - 1;
    memo.emplace(key, id);
    return id;
  }

  Ref constant(bool v) {
    NNode n;
    n.kind = GK_N_CONST;
    n.flags = 0;
    return Ref{intern_node("const0", n), v};
  }
  bool is_const(const Ref& r) const { return nodes[r.node].kind == GK_N_CONST; }
  bool const_val(const Ref& r) const { return r.neg; }   // the only CONST node holds 0

  int bcast(int node, int child_scope) {
    NNode n;
    n.kind = GK_N_BCAST;
    n.level = child_scope;
    n.scope = child_scope;
    n.a = node;
    return intern_node("bc" + std::to_string(node) + ">" + std::to_string(child_scope), n);
  }
  // bring a node up to a deeper level (target must be a descendant of the node's level)
  int raise(int node, int target) {
    int lvl = nodes[node].level;
    if (lvl == target) return node;
    std::vector<int> chain;
    for (int s = target; s != lvl; s = schema.scopes[s].parent) {
      if (s == 0) throw RegoError{"internal: netlist levels are not on one scope chain"};
      chain.push_back(s);
    }
    for (size_t i = chain.size(); i-- > 0;) node = bcast(node, chain[i]);
    return node;
  }

  // n-ary AND / OR over references of ONE level (after raising); folds constants, duplicates and x op !x
  Ref gate_n(bool is_or, std::vector<Ref> refs, int level) {
    std::vector<Ref> in;
    for (auto& r : refs) {
      if (is_const(r)) {
        bool cv = const_val(r);
        if (is_or == cv) return constant(is_or);   // x | 1 = 1 ; x & 0 = 0
        continue;                                  // x | 0 = x ; x & 1 = x
      }
      bool dup = false;
      for (auto& q : in)
        if (q.node == r.node) {
          if (q.neg != r.neg) return constant(is_or);
          dup = true;
        }
      if (!dup) in.push_back(r);
    }
    if (in.empty()) return constant(!is_or);
    if (in.size() == 1) return in[0];
    std::sort(in.begin(), in.end(), [](const Ref& p, const Ref& q) { return p.node != q.node ? p.node < q.node : p.neg < q.neg; });
    NNode n;
    n.kind = GK_N_GATE;
    n.level = level;
    n.flags = is_or ? GK_G_OR : 0;
    std::string key = is_or ? "or" : "and";
    for (auto& r : in) {
      n.ins.emplace_back(r.node, r.neg);
      key += (r.neg ? ",!" : ",") + std::to_string(r.node);
    }
    return Ref{intern_node(key, n), false};
  }

  // materialise a possibly negated reference as a plain node (needed where negation cannot be folded)
  int plain(Ref r) {
    if (!r.neg) return r.node;
    NNode n;
    n.kind = GK_N_GATE;
    n.level = nodes[r.node].level;
    n.ins.emplace_back(r.node, true);
    return intern_node("not" + std::to_string(r.node), n);
  }

  Ref build(const FP& f) {
    switch (f->k) {
      case Formula::True: return constant(true);
      case Formula::False: return constant(false);
      case Formula::Not: {
        Ref r = build(f->kids[0]);
        r.neg = !r.neg;
        return r;
      }
      case Formula::Atom: {
        NNode n;
        n.kind = GK_N_ATOM;
        n.level = schema.cols[f->col].scope;
        n.op = f->op;
        n.col = f->col;
        n.cval = f->cval;
        n.imm = f->imm;
        std::string key = "a" + std::to_string(f->op) + ":" + std::to_string(f->col) + ":" + std::to_string(f->imm) + ":" +
                          (f->cval ? intern_key(f->cval) : std::string());
        return Ref{intern_node(key, n), false};
      }
      case Formula::And:
      case Formula::Or: {
        std::vector<Ref> refs;
        for (auto& k : f->kids) refs.push_back(build(k));
        // one n-ary gate per level, shallow levels first: a loop-invariant group is broadcast into the loop once
        std::stable_sort(refs.begin(), refs.end(), [&](const Ref& p, const Ref& q) { return depth(nodes[p.node].level) < depth(nodes[q.node].level); });
        const bool is_or = f->k == Formula::Or;
        Ref acc = refs[0];
        size_t i = 1;
        while (true) {
          int lvl = nodes[acc.node].level;
          std::vector<Ref> group{acc};
          while (i < refs.size() && nodes[refs[i].node].level == lvl) group.push_back(refs[i++]);
          acc = gate_n(is_or, group, lvl);
          if (i >= refs.size()) break;
          // next group is deeper: raise the accumulated value into it
          int next = nodes[refs[i].node].level;
          if (!is_const(acc)) {
            if (depth(next) < depth(nodes[acc.node].level)) {   // constants sort first; keep the deeper level
              next = nodes[acc.node].level;
            }
            acc.node = raise(acc.node, next);
          }
          std::vector<Ref> g2{acc};
          while (i < refs.size() && nodes[refs[i].node].level == next) g2.push_back(refs[i++]);
          for (auto& r : g2)
            if (!is_const(r)) r.node = raise(r.node, next);
          acc = gate_n(is_or, g2, next);
          if (i >= refs.size()) break;
        }
        return acc;
      }
      case Formula::Exists: {
        Ref r = build(f->kids[0]);
        if (is_const(r)) {
          if (!const_val(r)) return constant(false);
          // EXISTS row: true  == the collection is non-empty: broadcast a constant 1 into the scope and OR-reduce it
        }
        int body = raise(plain(r), f->scope);
        if (nodes[body].level != f->scope) throw RegoError{"internal: EXISTS body is deeper than its scope"};
        NNode n;
        n.kind = f->two ? GK_N_ACC2 : GK_N_ACC;
        n.level = schema.scopes[f->scope].parent;
        n.scope = f->scope;
        n.a = body;
        return Ref{intern_node((f->two ? "acc2_" : "acc") + std::to_string(body) + "@" + std::to_string(f->scope), n), false};
      }
    }
    throw RegoError{"internal: unknown formula node"};
  }
};

}  // namespace

// E[s](A) | E[s](B) == E[s](A | B)   and   !E[s](A) & !E[s](B) == !E[s](A | B): fewer segmented reductions, and the
// OR happens on packed child-level words
static FP merge_exists(const FP& f) {
  if (f->kids.empty()) return f;
  std::vector<FP> kids;
  for (auto& k : f->kids) kids.push_back(merge_exists(k));
  if (f->k == Formula::Not) return f_not(kids[0]);
  if (f->k == Formula::Exists) return f->two ? f_exists2(f->scope, kids[0]) : f_exists(f->scope, kids[0]);
  const bool is_or = f->k == Formula::Or;
  std::map<int, std::vector<FP>> groups;
  std::vector<FP> rest;
  for (auto& k : kids) {
    if (is_or && k->k == Formula::Exists && !k->two) groups[k->scope].push_back(k->kids[0]);
    else if (!is_or && k->k == Formula::Not && k->kids[0]->k == Formula::Exists && !k->kids[0]->two) groups[k->kids[0]->scope].push_back(k->kids[0]->kids[0]);
    else rest.push_back(k);
  }
  FP out = is_or ? f_false() : f_true();
  for (auto& k : rest) out = is_or ? f_or(out, k) : f_and(out, k);
  for (auto& g : groups) {
    FP body = f_false();
    for (auto& b : g.second) body = f_or(body, b);
    FP e = f_exists(g.first, body);
    out = is_or ? f_or(out, e) : f_and(out, f_not(e));
  }
  return out;
}

// Nested independent iterations (`l := labels[k]; c := containers[_]; <test on c>; <test on l>`) lower to an EXISTS whose body
// mixes rows of two scopes that are not nested in each other.  The netlist only relates a scope to its ancestors, but a conjunct
// that does not depend on the inner loop can leave it:  E[s](A & B) == E[s](A) & B  when B has no row of s -- exact, also
// for an empty s (both sides false).
static bool on_chain(int level, int scope, const Schema& sc) {   // is `level` an ancestor-or-self of `scope`?
  for (int s = scope;; s = sc.scopes[s].parent) {
    if (s == level) return true;
    if (s == 0) return level == 0;
  }
}
// level at which the formula's value lives once built (deepest leaf after the reductions); -2: its leaves are not on one chain
static int formula_level(const FP& f, const Schema& sc) {
  switch (f->k) {
    case Formula::True:
    case Formula::False: return 0;
    case Formula::Atom: return sc.cols[f->col].scope;
    case Formula::Not: return formula_level(f->kids[0], sc);
    case Formula::Exists: {
      int b = formula_level(f->kids[0], sc);
      if (b == -2 || !on_chain(b, f->scope, sc)) return -2;
      return sc.scopes[f->scope].parent;
    }
    default: {
      int deepest = 0;
      for (auto& k : f->kids) {
        int l = formula_level(k, sc);
        if (l == -2) return -2;
        if (on_chain(deepest, l, sc)) deepest = l;
        else if (!on_chain(l, deepest, sc)) return -2;
      }
      return deepest;
    }
  }
}
static FP hoist_invariants(const FP& f, const Schema& sc) {
  if (f->kids.empty()) return f;
  std::vector<FP> kids;
  for (auto& k : f->kids) kids.push_back(hoist_invariants(k, sc));
  switch (f->k) {
    case Formula::Not: return f_not(kids[0]);
    case Formula::And: {
      FP out = f_true();
      for (auto& k : kids) out = f_and(out, k);
      return out;
    }
    case Formula::Or: {
      FP out = f_false();
      for (auto& k : kids) out = f_or(out, k);
      return out;
    }
    case Formula::Exists: {
      const FP& body = kids[0];
      std::vector<FP> conj = body->k == Formula::And ? body->kids : std::vector<FP>{body};
      FP inner = f_true(), outer = f_true();
      bool moved = false;
      for (auto& k : conj) {
        const int l = formula_level(k, sc);
        if (l != -2 && !on_chain(l, f->scope, sc)) {
          outer = f_and(outer, k);
          moved = true;
        } else {
          inner = f_and(inner, k);
        }
      }
      if (!moved) return f->two ? f_exists2(f->scope, body) : f_exists(f->scope, body);
      return f_and(f->two ? f_exists2(f->scope, inner) : f_exists(f->scope, inner), outer);
    }
    default: return f;
  }
}

// does the formula fit the netlist's scope tree?  (add_constraint asks before the constraint is accepted)
void check_netlist_shape(const FP& formula, const Schema& sc) {
  if (formula_level(hoist_invariants(formula, sc), sc) == -2)
    throw RegoError{"rego_unsupported: the rule iterates two unrelated collections in one body and tests them together in a way that cannot be "
                    "separated (a cross product); the GPU predicate table only nests a collection inside its parents"};
}

void NetBuilder::build(const std::vector<FP>& formulas, const std::vector<uint32_t>& match_id, uint32_t nmatch) {
  Net net(*schema);
  if (schema->scopes.size() > GK_MAX_SCOPES) throw RegoError{"rego_unsupported: too many iteration scopes"};
  // match nodes (+ a pseudo node that owns the error column's slot)
  std::vector<int> match_node(nmatch), err_node(nmatch);
  for (uint32_t m = 0; m < nmatch; ++m) {
    NNode e;
    e.kind = GK_N_CONST;   // placeholder kind; never emitted (flags = 2 marks it)
    e.flags = 2;
    err_node[m] = net.intern_node("err" + std::to_string(m), e);
    NNode n;
    n.kind = GK_N_MATCH;
    n.match_id = m;
    n.err_of = err_node[m];
    match_node[m] = net.intern_node("match" + std::to_string(m), n);
  }
  struct Out {
    int prog;
    uint32_t flags;
  };
  std::vector<Out> outs;
  for (auto& f : formulas) {
    Ref r = net.build(merge_exists(hoist_invariants(f, *schema)));
    Out o{-1, 0};
    if (net.is_const(r)) o.flags = net.const_val(r) ? 1u : 2u;
    else {
      o.prog = net.plain(r);
      if (net.nodes[o.prog].level != 0) throw RegoError{"internal: constraint result is not at the object level"};
    }
    outs.push_back(o);
  }
  auto& N = net.nodes;
  // ---- phases and liveness
  int maxphase = 0;
  for (auto& n : N) maxphase = std::max(maxphase, n.phase);
  const int out_phase = maxphase + 1;
  for (auto& n : N) n.last_use = n.phase;
  for (auto& n : N) {
    if (n.a >= 0) N[n.a].last_use = std::max(N[n.a].last_use, n.phase);
    if (n.b >= 0) N[n.b].last_use = std::max(N[n.b].last_use, n.phase);
    for (auto& in : n.ins) N[in.first].last_use = std::max(N[in.first].last_use, n.phase);
  }
  for (size_t c = 0; c < outs.size(); ++c) {
    if (outs[c].prog >= 0) N[outs[c].prog].last_use = out_phase;
    N[match_node[match_id[c]]].last_use = out_phase;
    N[err_node[match_id[c]]].last_use = out_phase;
  }
  // drop nodes nobody uses (e.g. the CONST node when every constant folded away)
  std::vector<bool> used(N.size(), false);
  for (size_t c = 0; c < outs.size(); ++c) {
    if (outs[c].prog >= 0) used[outs[c].prog] = true;
    used[match_node[match_id[c]]] = true;
    used[err_node[match_id[c]]] = true;
  }
  for (size_t i = N.size(); i-- > 0;) {
    if (!used[i]) continue;
    if (N[i].a >= 0) used[N[i].a] = true;
    if (N[i].b >= 0) used[N[i].b] = true;
    for (auto& in : N[i].ins) used[in.first] = true;
  }
  // ---- slot allocation: per level free lists, a slot is reusable in the phase after its last use
  std::vector<std::vector<int>> by_phase(out_phase + 1);
  for (size_t i = 0; i < N.size(); ++i)
    if (used[i]) by_phase[N[i].phase].push_back((int)i);
  std::map<int, std::vector<int>> free_slots;           // level -> slots
  std::vector<std::vector<int>> release_at(out_phase + 2);
  slot_level.clear();
  auto alloc = [&](int level) {
    auto& fl = free_slots[level];
    if (!fl.empty()) {
      int s = fl.back();
      fl.pop_back();
      return s;
    }
    if (slot_level.size() >= GK_MAX_SLOTS) throw RegoError{"rego_unsupported: netlist needs too many live columns"};
    slot_level.push_back((uint8_t)level);
    return (int)slot_level.size() - 1;
  };
  ops.clear();
  items.clear();
  phase_off.clear();
  n_nodes = n_atoms = n_gates = 0;
  // (cost, item) per phase: heavy work first so the dynamic scheduler packs the phase tightly
  auto flush_phase = [&](std::vector<std::pair<uint32_t, uint32_t>>& ph) {
    std::stable_sort(ph.begin(), ph.end(), [](auto& x, auto& y) { return x.first > y.first; });
    phase_off.push_back((uint32_t)items.size());
    for (auto& it : ph) items.push_back(it.second);
    ph.clear();
  };
  std::vector<std::pair<uint32_t, uint32_t>> cur_phase;
  auto add_item = [&](uint32_t cost, uint32_t nparts) {
    uint32_t ix = (uint32_t)ops.size();   // index of the op about to be pushed
    if (ix >= (1u << 20)) throw RegoError{"rego_unsupported: netlist too large"};
    for (uint32_t p2 = 0; p2 < nparts; ++p2) cur_phase.emplace_back(cost / nparts, ix | (p2 << 20) | (nparts << 26));
  };
  for (int ph = 0; ph <= maxphase; ++ph) {
    for (int s : release_at[ph]) free_slots[slot_level[s]].push_back(s);
    auto& ids = by_phase[ph];
    std::stable_sort(ids.begin(), ids.end(), [&](int x, int y) { return N[x].level < N[y].level; });
    for (int id : ids) {
      NNode& n = N[id];
      n.slot = alloc(n.level);
      release_at[std::min(n.last_use + 1, out_phase + 1)].push_back(n.slot);
    }
    std::map<int, std::vector<uint32_t>> acc_groups, bcast_groups, acc2_groups;   // scope -> (in slot | out slot << 16)
    struct ColAtoms {
      std::vector<GkOp> ops;
      uint32_t cost = 0;
      bool deep = false, heavy = false;
    };
    std::map<std::pair<int, int>, ColAtoms> col_atoms;               // (level, column) -> its atoms in this phase
    for (int id : ids) {
      NNode& n = N[id];
      ++n_nodes;
      if (n.kind == GK_N_ACC || n.kind == GK_N_BCAST || n.kind == GK_N_ACC2) {
        (n.kind == GK_N_ACC ? acc_groups : n.kind == GK_N_ACC2 ? acc2_groups : bcast_groups)[n.scope].push_back((uint32_t)N[n.a].slot | ((uint32_t)n.slot << 16));
        continue;
      }
      GkOp op{};
      const uint32_t out = (uint32_t)n.slot;
      switch (n.kind) {
        case GK_N_CONST:
          if (n.flags == 2) continue;   // error-column placeholder: written by its MATCH op
          op.w0 = GK_N_CONST | (0u << 8) | (out << 16);
          op.w1 = 0;
          break;
        case GK_N_MATCH:
          op.w0 = GK_N_MATCH | (0u << 8) | (out << 16);
          op.w1 = (uint32_t)N[n.err_of].slot;
          op.w2 = n.match_id;
          break;
        case GK_N_GATE:
          ++n_gates;
          op.w0 = GK_N_GATE | ((uint32_t)n.level << 8) | (out << 16);
          op.w1 = (uint32_t)pool.size();
          op.w2 = n.flags;
          op.w3 = (uint32_t)n.ins.size();
          for (auto& in : n.ins) pool.push_back((uint32_t)N[in.first].slot | (in.second ? 0x80000000u : 0u));
          break;
        case GK_N_ATOM: {
          ++n_atoms;
          uint32_t w2 = 0, w3 = 0;
          switch (n.op) {
            case GK_OP_TRUTHY:
            case GK_OP_DEFINED: break;
            case GK_OP_VTMASK: w2 = n.imm; break;
            case GK_OP_SID_EQ: w2 = interner->intern(intern_key(n.cval)); break;
            case GK_OP_SID_IN: {
              std::vector<uint32_t> ids2;
              for (auto& v : n.cval->items) ids2.push_back(interner->intern(intern_key(v)));
              std::sort(ids2.begin(), ids2.end());
              ids2.erase(std::unique(ids2.begin(), ids2.end()), ids2.end());
              w2 = (uint32_t)pool.size();
              w3 = (uint32_t)ids2.size();
              pool.insert(pool.end(), ids2.begin(), ids2.end());
              break;
            }
            case GK_OP_NUM_CMP: {
              const int64_t k = num_key(n.cval->n);   // (columns hold num_key(x) too)
              w2 = (uint32_t)pool.size();
              pool.push_back((uint32_t)((uint64_t)k & 0xffffffffu));
              pool.push_back((uint32_t)((uint64_t)k >> 32));
              w3 = n.imm;
              break;
            }
            case GK_OP_SUFFIX:
            case GK_OP_CONTAINS:
              w2 = add_bytes(n.cval->s);
              w3 = (uint32_t)n.cval->s.size();
              break;
            case GK_OP_ANYPREFIX: {
              std::vector<uint32_t> ent;
              for (auto& v : n.cval->items) {
                uint32_t h[GK_HEAD_WORDS] = {0, 0, 0, 0, 0, 0, 0, 0}, m[GK_HEAD_WORDS] = {0, 0, 0, 0, 0, 0, 0, 0};
                const size_t nb = std::min<size_t>(v->s.size(), GK_HEAD_BYTES);
                memcpy(h, v->s.data(), nb);
                memset(m, 0xff, nb);
                ent.push_back((uint32_t)v->s.size());
                ent.push_back(add_bytes(v->s));
                ent.insert(ent.end(), h, h + GK_HEAD_WORDS);
                ent.insert(ent.end(), m, m + GK_HEAD_WORDS);   // byte masks of the compared prefix
              }
              w2 = (uint32_t)pool.size();
              w3 = (uint32_t)n.cval->items.size();
              pool.insert(pool.end(), ent.begin(), ent.end());
              break;
            }
            case GK_OP_ANYSUFFIX: {
              std::vector<uint32_t> ent;
              for (auto& v : n.cval->items) {
                ent.push_back(add_bytes(v->s));
                ent.push_back((uint32_t)v->s.size());
              }
              w2 = (uint32_t)pool.size();
              w3 = (uint32_t)n.cval->items.size();
              pool.insert(pool.end(), ent.begin(), ent.end());
              break;
            }
            default: throw RegoError{"internal: unknown atom"};
          }
          op.w0 = GK_N_ATOM | ((uint32_t)n.level << 8) | (out << 16);
          op.w1 = (uint32_t)n.op | ((uint32_t)n.col << 8);
          op.w2 = w2;
          op.w3 = w3;
          break;
        }
        default: throw RegoError{"internal: unknown netlist node"};
      }
      {
        const bool deep = n.level != 0;
        uint32_t cost = 10, parts = 1;
        switch (n.kind) {
          case GK_N_MATCH: cost = 4000; parts = 4; break;
          case GK_N_ATOM:
            if (n.op >= GK_OP_PREFIX) { cost = deep ? 1200 : 600; parts = deep ? 4 : 2; }
            else if (n.op == GK_OP_SID_IN) cost = deep ? 300 : 150;
            else cost = deep ? 120 : 60;
            break;
          case GK_N_GATE: cost = (uint32_t)(8 + 4 * n.ins.size()) * (deep ? 2 : 1); break;
          case GK_N_BCAST:
          case GK_N_ACC2:
          case GK_N_ACC: cost = 200; break;
          default: break;
        }
        if (n.kind == GK_N_ATOM) {   // deferred: all atoms of a column become one op below
          ColAtoms& ca = col_atoms[{n.level, n.col}];
          ca.ops.push_back(op);
          ca.cost += cost;
          ca.deep = deep;
          ca.heavy = ca.heavy || n.op >= GK_OP_PREFIX;
          continue;
        }
        add_item(cost, parts);
      }
      ops.push_back(op);
    }
    for (auto& kv : col_atoms) {
      ColAtoms& ca = kv.second;
      // Atoms that test a row's type / sid / number (everything but the prefix / suffix / contains tests, which walk the 32-byte
      // HEAD record or the byte pool) CAN be fused per column: one GK_N_ATOMS op loads the column slice once per trip -- four
      // 32-row groups into registers -- and evaluates every atom of the column on them.  Fusing was slower than
      // one op per atom -- fewer instructions per atom, but 25 long items per tile balance worse over the CTA's 8 warps than
      // 100 short ones.  Off unless GK_FUSED_ATOMS=1.
      static const bool fuse = getenv("GK_FUSED_ATOMS") && atoi(getenv("GK_FUSED_ATOMS")) == 1;
      std::vector<GkOp> fused;
      for (auto& a : ca.ops) {
        const uint32_t aop = a.w1 & 0xffu;
        const bool heavy1 = aop >= GK_OP_PREFIX;
        if (fuse && !heavy1) {
          fused.push_back(a);
          continue;
        }
        const uint32_t cost1 = heavy1 ? (ca.deep ? 1200u : 600u) : aop == GK_OP_SID_IN ? (ca.deep ? 300u : 150u) : (ca.deep ? 120u : 60u);
        add_item(cost1, heavy1 ? (ca.deep ? 4u : 2u) : 1u);
        ops.push_back(a);
      }
      if (fused.size() == 1) {
        add_item(ca.deep ? 120u : 60u, 1u);
        ops.push_back(fused[0]);
      } else if (!fused.empty()) {
        while (pool.size() % 4) pool.push_back(0);   // entries are read with 128-bit loads
        GkOp op{};
        op.w0 = GK_N_ATOMS | ((uint32_t)kv.first.first << 8);
        op.w1 = (uint32_t)kv.first.second << 8;
        op.w2 = (uint32_t)pool.size();
        op.w3 = (uint32_t)fused.size();
        for (auto& a : fused) {
          pool.push_back((a.w1 & 0xffu) | (a.w0 & 0xffff0000u));   // atom op | out slot << 16
          pool.push_back(a.w2);
          pool.push_back(a.w3);
          pool.push_back(0);
        }
        const uint32_t cost = (ca.deep ? 100u : 50u) + (ca.deep ? 50u : 25u) * (uint32_t)fused.size();
        add_item(cost, ca.deep && fused.size() >= 4 ? 2u : 1u);
        ops.push_back(op);
      }
    }
    // every EXISTS (and every hoisted broadcast) over the same scope in this phase is ONE op: the child ranges and
    // their masks are computed once per parent row and applied to all (input, output) column pairs
    for (int pass = 0; pass < 3; ++pass)
      for (auto& g : pass == 0 ? acc_groups : pass == 1 ? bcast_groups : acc2_groups) {
        GkOp op{};
        op.w0 = (pass == 0 ? GK_N_ACC : pass == 1 ? GK_N_BCAST : GK_N_ACC2) | ((uint32_t)g.first << 8);
        op.w1 = (uint32_t)pool.size();
        op.w3 = (uint32_t)g.second.size();
        pool.insert(pool.end(), g.second.begin(), g.second.end());
        // a large EXISTS group is split by parent rows (finer splits measured slower); a broadcast zeroes its outputs
        // first: never split
        const uint32_t parts = (pass == 0 && g.second.size() > 8) ? 2u : 1u;
        add_item(150 + 30 * (uint32_t)g.second.size(), parts);
        ops.push_back(op);
      }
    flush_phase(cur_phase);
  }
  // the error placeholder slots must exist even if their phase-0 allocation happened above (it did)
  this->outs.clear();
  for (size_t c = 0; c < outs.size(); ++c) {
    GkOutEnt e{};
    e.prog_slot = outs[c].prog >= 0 ? (uint16_t)N[outs[c].prog].slot : (uint16_t)0;
    e.match_slot = (uint16_t)N[match_node[match_id[c]]].slot;
    e.err_slot = (uint16_t)N[err_node[match_id[c]]].slot;
    e.flags = (uint16_t)outs[c].flags;
    this->outs.push_back(e);
  }
  phase_off.push_back((uint32_t)items.size());
  ops.push_back(GkOp{GK_N_END, 0, 0, 0});
  n_phases = phase_off.size() - 1;
}

}  // namespace gk
