#include "engine.hpp"

#include <sched.h>

#include <deque>
#include <functional>

#include <chrono>

#include <algorithm>
#include <cstring>
#include <thread>
#include <stdexcept>

namespace gk {

// ============================================================================================ strings
StringTable::StringTable() {
  off_.push_back(0);
  // sid 0 = GK_SID_UNDEF, sid 1 = GK_SID_OTHER: reserved, empty bytes
  off_.push_back(0);
  off_.push_back(0);
  map_.reserve(1 << 16);
}
uint32_t StringTable::intern(const std::string& key) {
  {
    std::shared_lock<std::shared_mutex> l(mu_);
    auto it = map_.find(key);
    if (it != map_.end()) return it->second;
  }
  std::unique_lock<std::shared_mutex> l(mu_);
  auto it = map_.find(key);
  if (it != map_.end()) return it->second;
  uint32_t id = (uint32_t)off_.size() - 1;
  bytes_.insert(bytes_.end(), key.begin(), key.end());
  off_.push_back((uint32_t)bytes_.size());
  map_.emplace(key, id);
  n_.store((uint32_t)map_.size(), std::memory_order_relaxed);
  return id;
}
std::shared_ptr<const StringTable::Frozen> StringTable::freeze() {
  std::unique_lock<std::shared_mutex> l(mu_);
  if (!frozen_ || frozen_->size() != map_.size()) frozen_ = std::make_shared<const Frozen>(map_);
  return frozen_;
}
uint32_t StringTable::lookup(const std::string& key) const {
  std::shared_lock<std::shared_mutex> l(mu_);
  auto it = map_.find(key);
  return it == map_.end() ? GK_SID_UNDEF : it->second;
}
void StringTable::snapshot(std::vector<uint32_t>& off, std::vector<uint8_t>& bytes) const {
  std::shared_lock<std::shared_mutex> l(mu_);
  off = off_;
  bytes = bytes_;
}
uint32_t StringTable::size() const {
  std::shared_lock<std::shared_mutex> l(mu_);
  return (uint32_t)off_.size() - 1;
}
std::string StringTable::get(uint32_t sid) const {
  std::shared_lock<std::shared_mutex> l(mu_);
  if (sid + 1 >= off_.size()) return "";
  return std::string(bytes_.begin() + off_[sid], bytes_.begin() + off_[sid + 1]);
}

// ====================================================================================== small helpers
static std::string str_field(const VP& o, const char* k) {
  VP v = obj_get(o, k);
  return v && v->t == VT::Str ? v->s : std::string();
}
void split_gv(const VP& obj, std::string& group, std::string& version, std::string& kind) {
  std::string api = str_field(obj, "apiVersion");
  size_t p = api.find('/');
  if (p == std::string::npos) {
    group.clear();
    version = api;
  } else {
    group = api.substr(0, p);
    version = api.substr(p + 1);
  }
  kind = str_field(obj, "kind");
}
std::string meta_str(const VP& obj, const char* f) {
  VP md = obj_get(obj, "metadata");
  if (!md || md->t != VT::Obj) return "";
  return str_field(md, f);
}
// unstructured.GetLabels -> NestedStringMap: any non-string value makes the whole map unreadable
static const Node* labels_of(const VP& obj) {
  VP md = obj_get(obj, "metadata");
  if (!md || md->t != VT::Obj) return nullptr;
  VP ls = obj_get(md, "labels");
  if (!ls || ls->t != VT::Obj) return nullptr;
  for (auto& e : ls->kv)
    if (e.second->t != VT::Str) return nullptr;
  return ls.get();
}

static void parse_wildcard(const std::string& w, uint32_t& mode, std::string& lit) {
  // pkg/wildcard/wildcard.go:17-29
  bool pre = !w.empty() && w.front() == '*', suf = !w.empty() && w.back() == '*';
  if (pre && suf) {
    lit = w.substr(1);
    if (!lit.empty() && lit.back() == '*') lit.pop_back();
    mode = GK_W_CONTAINS;
  } else if (pre) {
    lit = w.substr(1);
    mode = GK_W_SUFFIX;
  } else if (suf) {
    lit = w.substr(0, w.size() - 1);
    mode = GK_W_PREFIX;
  } else {
    lit = w;
    mode = GK_W_EXACT;
  }
}

// k8s.io/apimachinery validation of label keys / values (restated; module not vendored)
static bool name_part_chars_ok(const std::string& s) {   // ([A-Za-z0-9][-A-Za-z0-9_.]*)?[A-Za-z0-9]
  if (s.empty()) return false;
  auto alnum = [](char c) { return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9'); };
  if (!alnum(s.front()) || !alnum(s.back())) return false;
  for (char c : s)
    if (!alnum(c) && c != '-' && c != '_' && c != '.') return false;
  return true;
}
static bool dns_subdomain_ok(const std::string& s) {      // the regex only; the length has its own message
  if (s.empty()) return false;
  size_t i = 0;
  while (i <= s.size()) {
    size_t j = s.find('.', i);
    if (j == std::string::npos) j = s.size();
    if (j == i) return false;
    for (size_t q = i; q < j; ++q) {
      char c = s[q];
      bool an = (c >= 'a' && c <= 'z') || (c >= '0' && c <= '9');
      if (!an && !(c == '-' && q != i && q + 1 != j)) return false;
    }
    i = j + 1;
  }
  return true;
}
// ---- label key / value validation with apimachinery's messages (util/validation IsQualifiedName, IsValidLabelValue)
static const char* kQNameMsg =
    "must consist of alphanumeric characters, '-', '_' or '.', and must start and end with an alphanumeric character "
    "(e.g. 'MyName',  or 'my.name',  or '123-abc', regex used for validation is '([A-Za-z0-9][-A-Za-z0-9_.]*)?[A-Za-z0-9]')";
static const char* kSubdomainMsg =
    "a lowercase RFC 1123 subdomain must consist of lower case alphanumeric characters, '-' or '.', and must start and end with "
    "an alphanumeric character (e.g. 'example.com', regex used for validation is "
    "'[a-z0-9]([-a-z0-9]*[a-z0-9])?(\\.[a-z0-9]([-a-z0-9]*[a-z0-9])?)*')";
static const char* kLabelValueMsg =
    "a valid label must be an empty string or consist of alphanumeric characters, '-', '_' or '.', and must start and end with "
    "an alphanumeric character (e.g. 'MyValue',  or 'my_value',  or '12345', regex used for validation is "
    "'(([A-Za-z0-9][-A-Za-z0-9_.]*)?[A-Za-z0-9])?')";

static std::vector<std::string> qualified_name_errors(const std::string& k) {
  std::vector<std::string> errs;
  size_t p = k.find('/');
  std::string name = k;
  if (p != std::string::npos) {
    if (k.find('/', p + 1) != std::string::npos)
      return {std::string("a qualified name ") + kQNameMsg + " with an optional DNS subdomain prefix and '/' (e.g. 'example.com/MyName')"};
    std::string prefix = k.substr(0, p);
    name = k.substr(p + 1);
    if (prefix.empty()) errs.push_back("prefix part must be non-empty");
    else {
      if (prefix.size() > 253) errs.push_back("prefix part must be no more than 253 characters");
      if (!dns_subdomain_ok(prefix)) errs.push_back(std::string("prefix part ") + kSubdomainMsg);
    }
  }
  if (name.empty()) errs.push_back("name part must be non-empty");
  else if (name.size() > 63) errs.push_back("name part must be no more than 63 characters");
  if (!name_part_chars_ok(name)) errs.push_back(std::string("name part ") + kQNameMsg);
  return errs;
}
static std::vector<std::string> label_value_errors(const std::string& v) {
  std::vector<std::string> errs;
  if (v.size() > 63) errs.push_back("must be no more than 63 characters");
  if (!v.empty() && !name_part_chars_ok(v)) errs.push_back(kLabelValueMsg);
  return errs;
}
static std::string join(const std::vector<std::string>& v, const char* sep) {
  std::string o;
  for (size_t i = 0; i < v.size(); ++i) {
    if (i) o += sep;
    o += v[i];
  }
  return o;
}
static std::string go_strings(const std::vector<std::string>& vals) {   // fmt %#v of a []string
  if (vals.empty()) return "[]string(nil)";
  std::string o = "[]string{";
  for (size_t i = 0; i < vals.size(); ++i) {
    if (i) o += ", ";
    json_quote(vals[i], o);
  }
  return o + "}";
}

struct SelReq {
  std::string key;
  uint32_t op;
  std::vector<std::string> vals;
};
// labels.NewRequirement: every problem of one requirement, aggregated as field.ErrorList.ToAggregate prints them
static std::string requirement_error(const SelReq& r) {
  std::vector<std::string> errs;
  auto ke = qualified_name_errors(r.key);
  std::string q;
  if (!ke.empty()) {
    q.clear();
    json_quote(r.key, q);
    errs.push_back("key: Invalid value: " + q + ": " + join(ke, "; "));
  }
  if ((r.op == GK_SEL_IN || r.op == GK_SEL_NOTIN) && r.vals.empty())
    errs.push_back("values: Invalid value: " + go_strings(r.vals) + ": for 'in', 'notin' operators, values set can't be empty");
  if ((r.op == GK_SEL_EXISTS || r.op == GK_SEL_NOTEXISTS) && !r.vals.empty())
    errs.push_back("values: Invalid value: " + go_strings(r.vals) + ": values set must be empty for exists and does not exist");
  for (size_t i = 0; i < r.vals.size(); ++i) {
    auto ve = label_value_errors(r.vals[i]);
    if (ve.empty()) continue;
    q.clear();
    json_quote(r.vals[i], q);
    errs.push_back("values[" + std::to_string(i) + "][" + r.key + "]: Invalid value: " + q + ": " + join(ve, "; "));
  }
  std::vector<std::string> uniq;
  for (auto& e : errs)
    if (std::find(uniq.begin(), uniq.end(), e) == uniq.end()) uniq.push_back(e);
  if (uniq.empty()) return "";
  return uniq.size() == 1 ? uniq[0] : "[" + join(uniq, ", ") + "]";
}
// metav1.LabelSelectorAsSelector: returns "" or the error text.  Requirements are built in order (matchLabels -- sorted
// here, a Go map there -- then matchExpressions); the first failing one is the error.
static std::string parse_selector(const VP& sel, std::vector<SelReq>& out) {
  if (!sel || sel->t != VT::Obj) return "";
  VP ml = obj_get(sel, "matchLabels");
  if (ml && ml->t == VT::Obj)
    for (auto& e : ml->kv) {
      SelReq r;
      r.key = e.first->s;
      r.op = GK_SEL_IN;
      r.vals.push_back(e.second->t == VT::Str ? e.second->s : fmt_value(e.second, true));
      std::string err = requirement_error(r);
      if (!err.empty()) return err;
      out.push_back(r);
    }
  VP me = obj_get(sel, "matchExpressions");
  if (me && me->t == VT::Arr)
    for (auto& x : me->items) {
      SelReq r;
      r.key = str_field(x, "key");
      std::string op = str_field(x, "operator");
      VP vals = obj_get(x, "values");
      if (vals && vals->t == VT::Arr)
        for (auto& v : vals->items) r.vals.push_back(v->t == VT::Str ? v->s : fmt_value(v, true));
      if (op == "In") r.op = GK_SEL_IN;
      else if (op == "NotIn") r.op = GK_SEL_NOTIN;
      else if (op == "Exists") r.op = GK_SEL_EXISTS;
      else if (op == "DoesNotExist") r.op = GK_SEL_NOTEXISTS;
      else return "\"" + op + "\" is not a valid label selector operator";
      std::string err = requirement_error(r);
      if (!err.empty()) return err;
      out.push_back(r);
    }
  return "";
}

// K8sValidationTarget.ValidateConstraint (pkg/target/target.go:178-214): spec.match.labelSelector / namespaceSelector must be
// maps, must convert to metav1.LabelSelector (types), and must pass apimachinery's ValidateLabelSelector.  Returns "" or the
// error text.  (The frameworks client calls this before Driver.AddConstraint; pinned by TestValidateConstraint.)
static const char* go_type_name(const VP& v) {
  switch (v->t) {
    case VT::Null: return "null";
    case VT::True:
    case VT::False: return "bool";
    case VT::Num: return "number";
    case VT::Str: return "string";
    case VT::Arr: return "array";
    default: return "object";
  }
}
static std::string selector_field_errors(const VP& sel, std::vector<std::string>& errs) {
  const std::string P = "spec.labelSelector";
  auto cannot = [&](const VP& v, const std::string& where) {
    return std::string("Could not convert JSON to LabelSelector: json: cannot unmarshal ") + go_type_name(v) + " into Go struct field " + where;
  };
  auto quote = [](const std::string& x) {
    std::string q;
    json_quote(x, q);
    return q;
  };
  VP ml = obj_get(sel, "matchLabels");
  if (ml && ml->t != VT::Null) {
    if (ml->t != VT::Obj) return cannot(ml, "LabelSelector.matchLabels of type map[string]string");
    for (auto& e : ml->kv)
      if (e.second->t != VT::Str) return cannot(e.second, "LabelSelector.matchLabels of type string");
  }
  VP me = obj_get(sel, "matchExpressions");
  if (me && me->t != VT::Null) {
    if (me->t != VT::Arr) return cannot(me, "LabelSelector.matchExpressions of type []v1.LabelSelectorRequirement");
    for (auto& x : me->items) {
      if (x->t != VT::Obj) return cannot(x, "LabelSelector.matchExpressions of type v1.LabelSelectorRequirement");
      for (const char* f : {"key", "operator"}) {
        VP v = obj_get(x, f);
        if (v && v->t != VT::Null && v->t != VT::Str) return cannot(v, std::string("LabelSelectorRequirement.matchExpressions.") + f + " of type string");
      }
      VP vals = obj_get(x, "values");
      if (vals && vals->t != VT::Null) {
        if (vals->t != VT::Arr) return cannot(vals, "LabelSelectorRequirement.matchExpressions.values of type []string");
        for (auto& v : vals->items)
          if (v->t != VT::Str) return cannot(v, "LabelSelectorRequirement.matchExpressions.values of type []string");
      }
    }
  }
  if (ml && ml->t == VT::Obj)
    for (auto& e : ml->kv) {   // (sorted by key)
      for (auto& m : qualified_name_errors(e.first->s)) errs.push_back(P + ".matchLabels: Invalid value: " + quote(e.first->s) + ": " + m);
      for (auto& m : label_value_errors(e.second->s)) errs.push_back(P + ".matchLabels: Invalid value: " + quote(e.second->s) + ": " + m);
    }
  if (me && me->t == VT::Arr)
    for (size_t i = 0; i < me->items.size(); ++i) {
      const VP& x = me->items[i];
      const std::string fp = P + ".matchExpressions[" + std::to_string(i) + "]";
      const std::string op = str_field(x, "operator"), key = str_field(x, "key");
      std::vector<std::string> vals;
      VP vs = obj_get(x, "values");
      if (vs && vs->t == VT::Arr)
        for (auto& v : vs->items) vals.push_back(v->s);
      if (op == "In" || op == "NotIn") {
        if (vals.empty()) errs.push_back(fp + ".values: Required value: must be specified when `operator` is 'In' or 'NotIn'");
      } else if (op == "Exists" || op == "DoesNotExist") {
        if (!vals.empty()) errs.push_back(fp + ".values: Forbidden: may not be specified when `operator` is 'Exists' or 'DoesNotExist'");
      } else {
        errs.push_back(fp + ".operator: Invalid value: " + quote(op) + ": not a valid selector operator");
      }
      for (auto& m : qualified_name_errors(key)) errs.push_back(fp + ".key: Invalid value: " + quote(key) + ": " + m);
      for (size_t j = 0; j < vals.size(); ++j)
        for (auto& m : label_value_errors(vals[j])) errs.push_back(fp + ".values[" + std::to_string(j) + "]: Invalid value: " + quote(vals[j]) + ": " + m);
    }
  return "";
}
// K8sValidationTarget.ToMatcher / convertToMatch (pkg/target/target.go:226-254): spec.match must be a map whose members have the
// JSON types of match.Match (pkg/mutation/match/match_types.go:13-51).  "" or the ErrCreatingMatcher text.
static std::string to_matcher_error(const VP& constraint) {
  VP spec = constraint && constraint->t == VT::Obj ? obj_get(constraint, "spec") : nullptr;
  VP m = spec && spec->t == VT::Obj ? obj_get(spec, "match") : nullptr;
  if (!m || m->t == VT::Null) return "";
  const std::string pre = "unable to create matcher: ";
  if (m->t != VT::Obj) return pre + ".spec.match accessor error: " + json_str(m) + " is of the type " + go_type_name(m) + ", expected map[string]interface{}";
  auto bad = [&](const VP& v, const std::string& field, const std::string& typ) {
    return pre + "could not convert JSON to Match: json: cannot unmarshal " + go_type_name(v) + " into Go struct field Match." + field + " of type " + typ;
  };
  auto strlist = [&](const VP& v, const std::string& field, const std::string& typ) -> std::string {
    if (!v || v->t == VT::Null) return "";
    if (v->t != VT::Arr) return bad(v, field, typ);
    for (auto& x : v->items)
      if (x->t != VT::Str) return bad(x, field, "string");
    return "";
  };
  for (const char* f : {"source", "scope", "name"}) {
    VP v = obj_get(m, f);
    if (v && v->t != VT::Null && v->t != VT::Str) return bad(v, f, "string");
  }
  VP kinds = obj_get(m, "kinds");
  if (kinds && kinds->t != VT::Null) {
    if (kinds->t != VT::Arr) return bad(kinds, "kinds", "[]match.Kinds");
    for (auto& k : kinds->items) {
      if (k->t != VT::Obj) return bad(k, "kinds", "match.Kinds");
      for (const char* f : {"apiGroups", "kinds"}) {
        std::string e = strlist(obj_get(k, f), std::string("kinds.") + f, "[]string");
        if (!e.empty()) return e;
      }
    }
  }
  for (const char* f : {"namespaces", "excludedNamespaces"}) {
    std::string e = strlist(obj_get(m, f), f, "[]wildcard.Wildcard");
    if (!e.empty()) return e;
  }
  for (const char* f : {"labelSelector", "namespaceSelector"}) {
    VP sel = obj_get(m, f);
    if (!sel || sel->t == VT::Null) continue;
    if (sel->t != VT::Obj) return bad(sel, f, "v1.LabelSelector");
    std::vector<std::string> ignored;
    std::string conv = selector_field_errors(sel, ignored);
    if (!conv.empty()) {
      const std::string from = "Could not convert JSON to LabelSelector";
      size_t at = conv.find(from);
      if (at != std::string::npos) conv.replace(at, from.size(), "could not convert JSON to Match");
      return pre + conv;
    }
  }
  return "";
}

std::string validate_constraint_json(const std::string& json) {
  VP cur;
  try {
    cur = json_parse(json.data(), json.size());
  } catch (JsonError& e) {
    return "invalid constraint: " + e.msg;
  }
  for (const char* part : {"spec", "match"}) {
    if (!cur || cur->t != VT::Obj) return "";
    cur = obj_get(cur, part);
    if (!cur) return "";
  }
  if (cur->t != VT::Obj) return ".spec.match accessor error: " + json_str(cur) + " is of the type " + go_type_name(cur) + ", expected map[string]interface{}";
  for (const char* f : {"labelSelector", "namespaceSelector"}) {
    VP sel = obj_get(cur, f);
    if (!sel || sel->t == VT::Null) continue;
    if (sel->t != VT::Obj)
      return std::string(".spec.match.") + f + " accessor error: " + json_str(sel) + " is of the type " + go_type_name(sel) + ", expected map[string]interface{}";
    std::vector<std::string> errs;
    std::string conv = selector_field_errors(sel, errs);
    if (!conv.empty()) return conv;
    std::vector<std::string> uniq;
    for (auto& e : errs)
      if (std::find(uniq.begin(), uniq.end(), e) == uniq.end()) uniq.push_back(e);
    if (!uniq.empty()) return uniq.size() == 1 ? uniq[0] : "[" + join(uniq, ", ") + "]";
  }
  return "";
}

// ============================================================================================== engine
// CPUs this process may actually use: the smaller of the affinity mask and the cgroup CPU quota (a container on a
// 128-thread host is often capped at a fraction of it; more runnable threads than quota only buys throttling).
int effective_cpus() {
  int n = (int)std::max(1u, std::thread::hardware_concurrency());
  cpu_set_t set;
  if (sched_getaffinity(0, sizeof set, &set) == 0) n = std::min(n, std::max(1, CPU_COUNT(&set)));
  auto quota = [&](const char* path_quota, const char* path_period) {
    FILE* f = fopen(path_quota, "r");
    if (!f) return;
    char a[64] = {0}, b[64] = {0};
    int got = fscanf(f, "%63s %63s", a, b);
    fclose(f);
    if (got < 1 || !strcmp(a, "max")) return;
    double q = atof(a), p = got >= 2 ? atof(b) : 0;
    if (path_period) {
      FILE* g = fopen(path_period, "r");
      if (g) {
        if (fscanf(g, "%63s", b) == 1) p = atof(b);
        fclose(g);
      }
    }
    if (q > 0 && p > 0) n = std::min(n, std::max(1, (int)(q / p + 0.5)));
  };
  quota("/sys/fs/cgroup/cpu.max", nullptr);                                                        // cgroup v2
  quota("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "/sys/fs/cgroup/cpu/cpu.cfs_period_us");          // cgroup v1
  return n;
}

Engine::Engine(int threads) : threads_(threads > 0 ? threads : effective_cpus()) {}

void Engine::add_template(const std::string& kind, const std::string& rego, const std::vector<std::string>& libs) {
  auto mod = rego_parse(rego, libs);   // throws RegoError on syntax / unsafe-var errors
  if (!mod->is_rule("violation")) throw RegoError{"rego_compile_error: template " + kind + " has no `violation` rule"};
  // lowering is parameter-specific, but unsupported constructs that do not depend on parameters surface
  // here: lower once against empty parameters and discard (errors that need parameters surface at AddConstraint)
  {
    Schema tmp;
    try {
      (void)lower_violation(mod, v_obj({}), tmp);
    } catch (RegoError& e) {
      if (e.msg.rfind("rego_unsupported", 0) == 0 || e.msg.rfind("rego_type_error", 0) == 0 || e.msg.rfind("rego_unsafe", 0) == 0) throw;
    }
  }
  std::unique_lock<std::shared_mutex> l(mu_);
  TemplateEntry t;
  t.kind = kind;
  t.src = rego;
  t.mod = mod;
  // replacing a template re-lowers its existing constraints with THEIR parameters: a replacement that no longer compiles for
  // them (or pushes the joint set over a limit) is rejected and the old template stays
  auto old = templates_.find(kind);
  const bool had = old != templates_.end();
  TemplateEntry prev;
  if (had) prev = old->second;
  templates_[kind] = std::move(t);
  bool used = false;
  for (auto& c : constraints_) used = used || c->kind == kind;
  if (used) {
    try {
      compile_locked();
    } catch (...) {
      if (had) templates_[kind] = prev;
      else templates_.erase(kind);
      dirty_ = true;
      throw;
    }
  } else {
    dirty_ = true;
  }
}

bool Engine::remove_template(const std::string& kind) {
  std::unique_lock<std::shared_mutex> l(mu_);
  bool had = templates_.erase(kind) != 0;
  // constraints of that kind go with it (the reference's client drops them with the template)
  constraints_.erase(std::remove_if(constraints_.begin(), constraints_.end(), [&](auto& c) { return c->kind == kind; }), constraints_.end());
  dirty_ = true;
  return had;
}

static std::string enforcement_action_of(const VP& obj) {
  // util.GetEnforcementAction -- pkg/util/enforcement_action.go:132-151
  VP spec = obj_get(obj, "spec");
  std::string ea = spec ? str_field(spec, "enforcementAction") : "";
  if (ea.empty()) return "deny";
  if (ea == "deny" || ea == "dryrun" || ea == "warn" || ea == "scoped") return ea;
  return "unrecognized";
}

void Engine::add_constraint(const std::string& json) {
  VP obj;
  try {
    obj = json_parse(json.data(), json.size());
  } catch (JsonError& e) {
    throw RegoError{"invalid constraint: " + e.msg};
  }
  if (obj->t != VT::Obj) throw RegoError{"invalid constraint: not an object"};
  auto c = std::make_shared<Constraint>();
  c->kind = str_field(obj, "kind");
  c->name = meta_str(obj, "name");
  if (c->kind.empty() || c->name.empty()) throw RegoError{"invalid constraint: kind and metadata.name are required"};
  c->obj = obj;
  {
    std::string terr = to_matcher_error(obj);
    if (!terr.empty()) throw RegoError{terr};
  }
  VP spec = obj_get(obj, "spec");
  VP params = spec ? obj_get(spec, "parameters") : nullptr;
  c->params = params && params->t != VT::Null ? params : v_obj({});
  c->params_key = json_str(c->params);
  c->action = enforcement_action_of(obj);
  if (spec) {
    VP sea = obj_get(spec, "scopedEnforcementActions");
    if (sea && sea->t == VT::Arr)
      for (auto& x : sea->items) {
        ScopedAction a;
        a.action = str_field(x, "action");
        VP eps = obj_get(x, "enforcementPoints");
        if (eps && eps->t == VT::Arr)
          for (auto& p : eps->items) a.points.push_back(str_field(p, "name"));
        c->scoped.push_back(a);
      }
    VP m = obj_get(spec, "match");
    if (m && m->t == VT::Obj) {
      c->match.has = true;
      c->match.raw = m;
    }
  }
  std::unique_lock<std::shared_mutex> l(mu_);
  auto tit = templates_.find(c->kind);
  if (tit == templates_.end()) throw RegoError{"no template registered for constraint kind " + c->kind};
  // lower now so that unsupported constructs are an AddConstraint error (like a Rego compile error)
  {
    Schema tmp;
    check_netlist_shape(lower_violation(tit->second.mod, c->params, tmp), tmp);
  }
  // The constraint set is compiled JOINTLY (one schema, one netlist): limits that only the whole set can hit -- iteration
  // scopes, columns, netlist size -- must fail THIS call, not every later review.  Trial-compile the prospective set and roll
  // the mutation back when it does not compile.
  auto saved = constraints_;
  bool replaced = false;
  for (auto& e : constraints_)
    if (e->kind == c->kind && e->name == c->name) {
      e = c;
      replaced = true;
    }
  if (!replaced) constraints_.push_back(c);
  try {
    compile_locked();
  } catch (...) {
    constraints_ = std::move(saved);
    dirty_ = true;
    throw;
  }
}

bool Engine::remove_constraint(const std::string& kind, const std::string& name) {
  std::unique_lock<std::shared_mutex> l(mu_);
  size_t before = constraints_.size();
  constraints_.erase(std::remove_if(constraints_.begin(), constraints_.end(), [&](auto& c) { return c->kind == kind && c->name == name; }),
                     constraints_.end());
  dirty_ = true;
  return constraints_.size() != before;
}

void Engine::put_namespace(const std::string& name, const std::string& json) {
  VP v;
  try {
    v = json_parse(json.data(), json.size());
  } catch (JsonError& e) {
    throw RegoError{"invalid namespace object: " + e.msg};
  }
  // nsCache.Add (pkg/target/ns_cache.go:22-44): a non-map is an error, a map that is not a core Namespace is ignored, a Namespace
  // that does not convert to corev1.Namespace (a member of the wrong JSON type) is an error
  if (v->t != VT::Obj) throw RegoError{std::string("cannot cache non-namespace type: cannot cache type ") + go_type_name(v) + ", want map[string]interface {}"};
  {
    std::string g, ver, k;
    split_gv(v, g, ver, k);
    if (k != "Namespace" || !g.empty()) return;
  }
  auto is_obj_or_absent = [](const VP& x) { return !x || x->t == VT::Null || x->t == VT::Obj; };
  VP md = obj_get(v, "metadata");
  bool ok = is_obj_or_absent(md) && is_obj_or_absent(obj_get(v, "spec")) && is_obj_or_absent(obj_get(v, "status"));
  if (ok && md && md->t == VT::Obj) {
    for (const char* f : {"labels", "annotations"}) {
      VP ls = obj_get(md, f);
      ok = ok && is_obj_or_absent(ls);
      if (ok && ls && ls->t == VT::Obj)
        for (auto& e : ls->kv) ok = ok && e.second->t == VT::Str;
    }
    VP nm = obj_get(md, "name");
    ok = ok && (!nm || nm->t == VT::Null || nm->t == VT::Str);
  }
  if (!ok) throw RegoError{"cannot cache non-namespace type: cannot cache Namespace: <nil>"};
  std::unique_lock<std::shared_mutex> l(mu_);
  namespaces_[name] = v;
  ++ns_version_;
}
bool Engine::remove_namespace(const std::string& name) {
  std::unique_lock<std::shared_mutex> l(mu_);
  ++ns_version_;
  return namespaces_.erase(name) != 0;
}

// processUnstructured -- pkg/target/target.go:40-57
static std::vector<std::string> inventory_path(const VP& v) {
  if (!v || v->t != VT::Obj) throw RegoError{"unrecognized type, got " + std::string(v ? go_type_name(v) : "<nil>")};
  std::string g, ver, k;
  split_gv(v, g, ver, k);
  const std::string name = meta_str(v, "name"), ns = meta_str(v, "namespace");
  if (ver.empty()) throw RegoError{"invalid request object: resource " + name + " has no version"};
  if (k.empty()) throw RegoError{"invalid request object: resource " + name + " has no kind"};
  const std::string gv = g.empty() ? ver : g + "/" + ver;
  if (ns.empty()) return {"cluster", gv, k, name};
  return {"namespace", ns, gv, k, name};
}

std::vector<std::string> Engine::data_path(const std::string& json) {
  try {
    return inventory_path(json_parse(json.data(), json.size()));
  } catch (JsonError& e) {
    throw RegoError{"invalid data object: " + e.msg};
  }
}

void Engine::add_data(const std::vector<std::string>& path, const std::string& json) {
  VP v;
  try {
    v = json_parse(json.data(), json.size());
  } catch (JsonError& e) {
    throw RegoError{"invalid data object: " + e.msg};
  }
  std::vector<std::string> p = path.empty() ? inventory_path(v) : path;
  std::unique_lock<std::shared_mutex> l(mu_);
  inventory_[std::move(p)] = v;
  ++inventory_version_;
}

bool Engine::remove_data(const std::vector<std::string>& path) {
  std::unique_lock<std::shared_mutex> l(mu_);
  ++inventory_version_;
  // a path names one object or a whole sub-tree (storage.RemoveData on an inner node)
  bool any = false;
  for (auto it = inventory_.begin(); it != inventory_.end();) {
    const auto& k = it->first;
    if (k.size() >= path.size() && std::equal(path.begin(), path.end(), k.begin())) {
      it = inventory_.erase(it);
      any = true;
    } else {
      ++it;
    }
  }
  return any;
}

VP Engine::data_doc(uint64_t* version) {
  std::unique_lock<std::shared_mutex> l(mu_);
  if (!inventory_doc_ || inventory_doc_version_ != inventory_version_) {
    // the paths are sorted: children of one prefix are adjacent
    using It = std::map<std::vector<std::string>, VP>::const_iterator;
    std::function<VP(It, It, size_t)> build = [&](It lo, It hi, size_t depth) -> VP {
      std::vector<std::pair<VP, VP>> kv;
      while (lo != hi) {
        const std::string& key = lo->first[depth];
        It e = lo;
        while (e != hi && e->first[depth] == key) ++e;
        if (lo->first.size() == depth + 1) kv.emplace_back(v_str(key), lo->second);
        else kv.emplace_back(v_str(key), build(lo, e, depth + 1));
        lo = e;
      }
      return v_obj(std::move(kv));
    };
    inventory_doc_ = v_obj({{v_str("inventory"), build(inventory_.begin(), inventory_.end(), 0)}});
    inventory_doc_version_ = inventory_version_;
  }
  if (version) *version = inventory_version_;
  return inventory_doc_;
}

std::vector<std::string> scoped_actions_for(const Constraint& c, const std::string& ep) {
  std::vector<std::string> out;
  for (auto& a : c.scoped)
    for (auto& p : a.points)
      if (p == ep || p == "*") {
        out.push_back(a.action);
        break;
      }
  return out;
}

void Engine::active_mask(const Compiled& c, const std::string& ep, std::vector<uint32_t>& active) const {
  active.assign(c.order.size(), 1);
  for (size_t i = 0; i < c.order.size(); ++i)
    if (c.order[i]->action == "scoped" && scoped_actions_for(*c.order[i], ep).empty()) active[i] = 0;
}

// ---------------------------------------------------------------------------------------------- compile
std::shared_ptr<const Compiled> Engine::compiled() {
  {
    std::shared_lock<std::shared_mutex> l(mu_);
    if (!dirty_ && compiled_) return compiled_;
  }
  std::unique_lock<std::shared_mutex> l(mu_);
  if (dirty_ || !compiled_) compile_locked();
  return compiled_;
}

void Engine::compile_locked() {
  auto out = std::make_shared<Compiled>();
  out->version = ++version_;
  NetBuilder pb;
  pb.interner = &strings_;
  pb.schema = &out->schema;
  // pass 1: lower every constraint (fills the shared schema); group constraints that share a match block so the
  // kernel evaluates each distinct spec.match once per object
  std::vector<Constraint*> live;
  std::vector<FP> live_formula;
  std::vector<uint8_t> live_single;
  std::vector<FP> live_amb;
  std::map<std::string, uint32_t> match_ix;
  std::vector<uint32_t> mid_of;
  // First choice: every constraint lowered for the DEVICE INGEST path (all scopes / columns computable by the ingest kernels
  // from the raw JSON).  If one constraint cannot be, the whole set is lowered the classic way (maximal host closures) and
  // batches of this snapshot are flattened on the host.
  auto lower_all = [&](bool device_mode) {
    out->schema = Schema();
    out->pins.clear();
    live.clear();
    live_formula.clear();
    live_single.clear();
    live_amb.clear();
    match_ix.clear();
    mid_of.clear();
    for (auto& cp : constraints_) {
      Constraint& c = *cp;
      out->pins.push_back(cp);
      auto tit = templates_.find(c.kind);
      if (tit == templates_.end()) continue;
      bool single = false;
      FP amb;
      live_formula.push_back(lower_violation(tit->second.mod, c.params, out->schema, device_mode, &single, &amb));
      live_single.push_back(single ? 1 : 0);
      live_amb.push_back(amb);
      std::string key = c.match.has ? json_str(c.match.raw) : std::string();
      auto it = match_ix.find(key);
      uint32_t mid = it == match_ix.end() ? (uint32_t)match_ix.size() : it->second;
      if (it == match_ix.end()) match_ix.emplace(key, mid);
      live.push_back(&c);
      mid_of.push_back(mid);
    }
    out->schema.device_only = false;
  };
  static const bool no_device = getenv("GK_NO_DEVICE_INGEST") != nullptr;
  bool device_ok = !no_device;
  if (device_ok) {
    try {
      lower_all(true);
      device_ok = schema_device_ingestable(out->schema, &out->host_ingest_reason);
      if (device_ok) out->xprog = build_xprog(out->schema);
    } catch (RegoError& e) {
      if (e.msg.find("rego_unsupported") == std::string::npos) throw;
      device_ok = false;
      out->host_ingest_reason = e.msg;
    }
  }
  if (!device_ok) lower_all(false);
  out->device_ingest = device_ok;
  out->uses_data = out->schema.uses_data;
  std::vector<size_t> perm(live.size());
  for (size_t i = 0; i < perm.size(); ++i) perm[i] = i;
  std::stable_sort(perm.begin(), perm.end(), [&](size_t a, size_t b) { return mid_of[a] < mid_of[b]; });
  std::vector<FP> all, all_amb;
  for (size_t i : perm) {
    all_amb.push_back(live_amb[i]);
    out->order.push_back(live[i]);
    out->mods.push_back(templates_.at(live[i]->kind).mod);
    all.push_back(live_formula[i]);
    out->formulas.push_back(live_formula[i]);
    out->single_result.push_back(live_single[i]);
    out->cons_match.push_back(mid_of[i]);
  }
  out->match.resize(match_ix.size());
  std::vector<bool> built(match_ix.size(), false);
  // pass 2: emit code + match blocks
  for (size_t oi = 0; oi < perm.size(); ++oi) {
    Constraint& c = *live[perm[oi]];
    const uint32_t mid = mid_of[perm[oi]];
    GkMatch m{};
    MatchSpec ms = c.match;   // (a copy: the error texts below go into the snapshot)
    ms.lsel_err.clear();
    ms.nssel_err.clear();
    ms.src_err.clear();
    if (ms.has) {
      m.flags |= GK_M_HAS_MATCH;
      const VP& r = ms.raw;
      const bool emit_pool = !built[mid];   // pool entries are written once per distinct block
      VP kinds = obj_get(r, "kinds");
      if (emit_pool && kinds && kinds->t == VT::Arr && !kinds->items.empty()) {
        m.kinds_off = (uint32_t)pb.pool.size();
        for (auto& e : kinds->items) {
          std::vector<uint32_t> ks, gs;
          uint32_t wild = 0;
          VP kk = obj_get(e, "kinds"), gg = obj_get(e, "apiGroups");
          if (kk && kk->t == VT::Arr)
            for (auto& x : kk->items) {
              std::string s = x->t == VT::Str ? x->s : "";
              if (s == "*") wild |= 1;
              ks.push_back(strings_.intern("s" + s));
            }
          if (gg && gg->t == VT::Arr)
            for (auto& x : gg->items) {
              std::string s = x->t == VT::Str ? x->s : "";
              if (s == "*") wild |= 2;
              gs.push_back(strings_.intern("s" + s));
            }
          pb.pool.push_back((uint32_t)ks.size());
          pb.pool.push_back((uint32_t)gs.size());
          pb.pool.push_back(wild);
          pb.pool.insert(pb.pool.end(), ks.begin(), ks.end());
          pb.pool.insert(pb.pool.end(), gs.begin(), gs.end());
          ++m.kinds_n;
        }
      }
      std::string scope = str_field(r, "scope");
      if (scope == "Cluster") m.flags |= GK_M_SCOPE_CLUSTER;
      else if (scope == "Namespaced") m.flags |= GK_M_SCOPE_NAMESPACED;
      auto wild_list = [&](const char* field, uint32_t& off, uint32_t& n) {
        VP l = obj_get(r, field);
        if (!emit_pool || !l || l->t != VT::Arr) return;
        off = (uint32_t)pb.pool.size();
        for (auto& x : l->items) {
          uint32_t mode;
          std::string lit;
          parse_wildcard(x->t == VT::Str ? x->s : "", mode, lit);
          pb.pool.push_back(mode);
          pb.pool.push_back(pb.add_bytes(lit));
          pb.pool.push_back((uint32_t)lit.size());
          ++n;
        }
      };
      wild_list("namespaces", m.ns_off, m.ns_n);
      wild_list("excludedNamespaces", m.exns_off, m.exns_n);
      auto selector = [&](const char* field, uint32_t has_flag, uint32_t bad_flag, uint32_t& off, uint32_t& n, std::string& err) {
        VP s = obj_get(r, field);
        if (!s || s->t == VT::Null) return;
        m.flags |= has_flag;
        std::vector<SelReq> reqs;
        err = parse_selector(s, reqs);
        if (!err.empty()) {
          m.flags |= bad_flag;
          return;
        }
        if (!emit_pool) return;
        off = (uint32_t)pb.pool.size();
        for (auto& q : reqs) {
          pb.pool.push_back(strings_.intern("s" + q.key));
          pb.pool.push_back(q.op);
          pb.pool.push_back((uint32_t)q.vals.size());
          for (auto& v : q.vals) pb.pool.push_back(strings_.intern("s" + v));
          ++n;
        }
      };
      selector("labelSelector", GK_M_HAS_LSEL, GK_M_LSEL_INVALID, m.lsel_off, m.lsel_n, ms.lsel_err);
      selector("namespaceSelector", GK_M_HAS_NSSEL, GK_M_NSSEL_INVALID, m.nssel_off, m.nssel_n, ms.nssel_err);
      std::string name = str_field(r, "name");
      if (!name.empty()) {
        m.flags |= GK_M_HAS_NAME;
        std::string lit;
        parse_wildcard(name, m.name_mode, lit);
        if (emit_pool) m.name_boff = pb.add_bytes(lit);
        m.name_len = (uint32_t)lit.size();
      }
      std::string src = str_field(r, "source");
      uint32_t code = GK_SRC_ALL;
      if (src.empty() || src == "All") code = GK_SRC_ALL;
      else if (src == "Original") code = GK_SRC_ORIGINAL;
      else if (src == "Generated") code = GK_SRC_GENERATED;
      else {
        m.flags |= GK_M_SRC_INVALID;
        ms.src_err = "invalid source field \"" + src + "\"";
      }
      m.flags |= code << GK_M_SRC_SHIFT;
    }
    if (!built[mid]) {
      out->match[mid] = m;
      built[mid] = true;
    }
    out->match_errs.push_back(Compiled::MatchErrs{ms.lsel_err, ms.nssel_err, ms.src_err});
  }
  if (out->match.empty()) out->match.push_back(GkMatch{});
  // the audit's ambiguity netlist (same schema, same match blocks): output c is false only where constraint c has at most one
  // result for the object -- built from the pool / constant bytes as they stand before the decision netlist is appended
  NetBuilder pb2;
  pb2.interner = &strings_;
  pb2.schema = &out->schema;
  pb2.pool = pb.pool;
  pb2.cbytes = pb.cbytes;
  pb.build(all, out->cons_match, (uint32_t)match_ix.size());
  out->ops = std::move(pb.ops);
  out->items = std::move(pb.items);
  out->phase_off = std::move(pb.phase_off);
  out->outs = std::move(pb.outs);
  out->slot_level = std::move(pb.slot_level);
  out->pool = std::move(pb.pool);
  out->cbytes = std::move(pb.cbytes);
  if (out->pool.empty()) out->pool.push_back(0);
  if (out->cbytes.empty()) out->cbytes.push_back(0);
  if (out->slot_level.empty()) out->slot_level.push_back(0);
  out->n_nodes = pb.n_nodes;
  out->n_atoms = pb.n_atoms;
  out->n_gates = pb.n_gates;
  out->n_phases = pb.n_phases;
  if (std::any_of(out->single_result.begin(), out->single_result.end(), [](uint8_t x) { return x == 0; })) {
    try {
      for (auto& f : all_amb) check_netlist_shape(f, out->schema);
      pb2.build(all_amb, out->cons_match, (uint32_t)match_ix.size());
      auto amb = std::make_shared<Compiled>(*out);
      amb->version = ++version_;
      amb->formulas = all_amb;
      amb->ops = std::move(pb2.ops);
      amb->items = std::move(pb2.items);
      amb->phase_off = std::move(pb2.phase_off);
      amb->outs = std::move(pb2.outs);
      amb->slot_level = std::move(pb2.slot_level);
      amb->pool = std::move(pb2.pool);
      amb->cbytes = std::move(pb2.cbytes);
      if (amb->pool.empty()) amb->pool.push_back(0);
      if (amb->cbytes.empty()) amb->cbytes.push_back(0);
      if (amb->slot_level.empty()) amb->slot_level.push_back(0);
      amb->n_nodes = pb2.n_nodes, amb->n_atoms = pb2.n_atoms, amb->n_gates = pb2.n_gates, amb->n_phases = pb2.n_phases;
      out->amb = amb;
    } catch (RegoError&) {
      out->amb = nullptr;   // (a shape the netlist cannot hold: the audit evaluates every pair of the multi-result constraints)
    }
  }
  compiled_ = out;
  dirty_ = false;
}

std::string Engine::dump() {
  auto c = compiled();
  static const char* kXK[] = {"host", "path", "elem", "key", "count", "lut"};
  std::string o = "schema: " + std::to_string(c->schema.scopes.size() - 1) + " scopes, " + std::to_string(c->schema.cols.size()) +
                  " columns; netlist: " + std::to_string(c->n_nodes) + " nodes (" + std::to_string(c->n_atoms) + " atoms, " +
                  std::to_string(c->n_gates) + " gates) in " + std::to_string(c->n_phases) + " phases, " + std::to_string(c->slot_level.size()) +
                  " live slots, " + std::to_string(c->match.size()) + " distinct match blocks\n";
  o += c->device_ingest ? "  ingest: device (every scope / column is computed from the raw JSON by the ingest kernels)\n"
                        : "  ingest: host flattener (" + c->host_ingest_reason + ")\n";
  {
    std::vector<int> per(c->schema.scopes.size(), 0);
    for (uint8_t l : c->slot_level) per[l]++;
    o += "  slots per scope:";
    for (size_t i = 0; i < per.size(); ++i) o += " s" + std::to_string(i) + "=" + std::to_string(per[i]);
    o += "; items per phase:";
    for (size_t i = 0; i + 1 < c->phase_off.size(); ++i) o += " " + std::to_string(c->phase_off[i + 1] - c->phase_off[i]);
    o += "\n";
  }
  {
    // op mix: per kind and level, the number of ops and of (input, output) pairs / gate inputs / atoms per column
    std::map<std::string, std::pair<int, int>> mix;
    std::map<uint32_t, int> atoms_per_col;
    for (auto& op : c->ops) {
      uint32_t kind = op.w0 & 0xff, level = (op.w0 >> 8) & 0xff;
      const char* nm = kind == GK_N_ATOM ? "atom" : kind == GK_N_GATE ? "gate" : kind == GK_N_BCAST ? "bcast" : kind == GK_N_ACC ? "acc" : kind == GK_N_ACC2 ? "acc2"
                       : kind == GK_N_MATCH ? "match" : kind == GK_N_CONST ? "const" : kind == GK_N_ATOMS ? "atoms" : kind == GK_N_END ? "end" : "?";
      auto& m = mix[std::string(nm) + "@s" + std::to_string(level)];
      m.first++;
      m.second += (kind == GK_N_GATE || kind == GK_N_BCAST || kind == GK_N_ACC || kind == GK_N_ACC2 || kind == GK_N_ATOMS) ? (int)op.w3 : 1;
      if (kind == GK_N_ATOM) atoms_per_col[op.w1 >> 8]++;
      if (kind == GK_N_ATOMS) atoms_per_col[op.w1 >> 8] += (int)op.w3;
    }
    o += "  op mix (ops/operands):";
    for (auto& kv : mix) o += " " + kv.first + "=" + std::to_string(kv.second.first) + "/" + std::to_string(kv.second.second);
    o += "\n  atoms per column:";
    for (auto& kv : atoms_per_col) o += " c" + std::to_string(kv.first) + "=" + std::to_string(kv.second);
    o += "\n";
  }
  for (size_t i = 1; i < c->schema.scopes.size(); ++i)
    o += "  scope " + std::to_string(i) + " parent " + std::to_string(c->schema.scopes[i].parent) + ": " + c->schema.scopes[i].gen->key + "\n";
  for (size_t i = 0; i < c->schema.cols.size(); ++i)
    o += "  col " + std::to_string(i) + " scope " + std::to_string(c->schema.cols[i].scope) + " enc " + std::to_string(c->schema.cols[i].enc) + " " +
         std::string(kXK[(int)closure_xinfo(*c->schema.cols[i].expr).k]) + ": " + c->schema.cols[i].expr->key + "\n";
  for (size_t i = 0; i < c->order.size(); ++i)
    o += "constraint " + std::to_string(i) + " " + c->order[i]->kind + "/" + c->order[i]->name + (c->single_result[i] ? " [one result per pair]" : "") + ": " +
         formula_str(c->formulas[i], c->schema) + "\n";
  return o;
}

// ------------------------------------------------------------------------------------------- review doc
VP Engine::review_doc(const ObjIn& in, VP* obj_out, VP* old_out, VP* ns_out, std::string* err, const std::map<std::string, VP>* ns_snapshot) {
  VP obj, old, ns;
  auto parse = [&](const char* p, size_t n, const char* what, VP& dst) -> bool {
    if (!p) return true;
    try {
      dst = json_parse(p, n);
    } catch (JsonError& e) {
      *err = std::string("invalid request object: failed to unmarshal gkReview ") + what + ": " + e.msg;
      return false;
    }
    if (dst->t == VT::Null) {
      dst = nullptr;
      return true;
    }
    if (dst->t != VT::Obj) {
      *err = std::string("invalid request object: ") + what + " is not a JSON object";
      return false;
    }
    if (str_field(dst, "kind").empty()) {
      *err = std::string("invalid request object: failed to unmarshal gkReview ") + what + ": Object 'Kind' is missing";
      return false;
    }
    return true;
  };
  if (!parse(in.json, in.len, "object", obj) || !parse(in.old_json, in.old_len, "oldObject", old)) return nullptr;
  if (in.ns_json) {
    try {
      ns = json_parse(in.ns_json, in.ns_len);
      if (ns->t != VT::Obj) ns = nullptr;
    } catch (JsonError& e) {
      *err = "invalid namespace object: " + e.msg;
      return nullptr;
    }
  }
  std::string op = in.operation ? in.operation : "";
  if (op == "DELETE") {   // setObjectOnDelete -- pkg/target/target.go:262-280
    if (!old) {
      *err = "oldObject cannot be nil for DELETE operations";
      return nullptr;
    }
    obj = old;
  }
  VP ref = obj ? obj : old;
  std::string g, v, k, name, nsname;
  if (ref) {
    split_gv(ref, g, v, k);
    name = meta_str(ref, "name");
    nsname = meta_str(ref, "namespace");
  }
  if (in.ns_name) nsname = in.ns_name;
  VP user;
  if (in.userinfo_json) {
    try {
      user = json_parse(in.userinfo_json, in.userinfo_len);
    } catch (JsonError&) {
    }
  }
  // keys and constant members are per-thread singletons: the document is rebuilt for every object
  struct Keys {
    VP uid = v_str("uid"), kind = v_str("kind"), resource = v_str("resource"), operation = v_str("operation"), userInfo = v_str("userInfo"),
       object = v_str("object"), oldObject = v_str("oldObject"), options = v_str("options"), name = v_str("name"), ns = v_str("namespace"),
       nsobj = v_str("namespaceObject"), group = v_str("group"), version = v_str("version"), empty = v_str(""),
       no_resource = v_obj({{v_str("group"), v_str("")}, {v_str("version"), v_str("")}, {v_str("resource"), v_str("")}}), no_user = v_obj({});
  };
  static thread_local Keys K;
  if (!user) user = K.no_user;
  std::vector<std::pair<VP, VP>> kv;
  kv.reserve(11);
  // (already in key order: v_obj's sort has nothing to move)
  kv.emplace_back(K.kind, v_obj({{K.group, v_str(g)}, {K.kind, v_str(k)}, {K.version, v_str(v)}}));
  if (!name.empty()) kv.emplace_back(K.name, v_str(name));
  if (!nsname.empty()) kv.emplace_back(K.ns, v_str(nsname));
  if (ns) kv.emplace_back(K.nsobj, ns);
  kv.emplace_back(K.object, obj ? obj : v_null());
  kv.emplace_back(K.oldObject, old ? old : v_null());
  kv.emplace_back(K.operation, op.empty() ? K.empty : v_str(op));
  kv.emplace_back(K.options, v_null());
  kv.emplace_back(K.resource, K.no_resource);
  kv.emplace_back(K.uid, K.empty);
  kv.emplace_back(K.userInfo, user);
  if (obj_out) *obj_out = obj;
  if (old_out) *old_out = old;
  if (ns_out) {
    // Matcher.Match: review's namespace object, else the cache entry for review.Namespace (matcher.go:37-39)
    if (!ns && !nsname.empty()) {
      if (ns_snapshot) {   // flatten workers use a private copy: no lock traffic per object
        auto it = ns_snapshot->find(nsname);
        if (it != ns_snapshot->end()) ns = it->second;
      } else {
        std::shared_lock<std::shared_mutex> l(mu_);
        auto it = namespaces_.find(nsname);
        if (it != namespaces_.end()) ns = it->second;
      }
    }
    *ns_out = ns;
  }
  return v_obj(std::move(kv));
}

// =========================================================================================== flatten
// Wildcard.Matches -- pkg/wildcard/wildcard.go:17-30 (host copy for the excluder stage; the matcher's runs on the device)
static bool wildcard_match(const std::string& pat, const std::string& s) {
  bool pre = !pat.empty() && pat.front() == '*', suf = pat.size() > (pre ? 1u : 0u) && pat.back() == '*';
  if (pat == "*") return true;
  std::string core = pat.substr(pre ? 1 : 0, pat.size() - (pre ? 1 : 0) - (suf ? 1 : 0));
  if (pre && suf) return s.find(core) != std::string::npos;
  if (pre) return s.size() >= core.size() && s.compare(s.size() - core.size(), core.size(), core) == 0;
  if (suf) return s.compare(0, core.size(), core) == 0;
  return s == pat;
}
// What one chunk of objects flattens to; chunks are merged in object order afterwards.
struct ChunkOut {
  HostBatch hb;
  // old-object header rows are kept in a second set of vectors and appended after the merge
  std::vector<uint32_t> o_flags, o_kind, o_group, o_nsn_off{0}, o_name_off{0}, o_gen_off{0}, o_lbl_off{0}, o_lbl_kv;
  std::vector<uint8_t> o_name_bytes, o_gen_bytes, o_nsn_bytes;
  bool any_old = false;
};

struct Flattener : ChunkOut {
  Engine& eng;
  const Compiled& c;
  std::unordered_map<std::string, uint32_t> sid_cache;
  std::unordered_map<const Module*, std::unique_ptr<Eval>> evals;
  std::vector<VP> ns_objs;                             // namespace table rows of this chunk
  std::unordered_map<const Node*, uint32_t> ns_row_of;

  struct Row {
    VP elem, key;
    uint32_t parent;
  };
  std::vector<std::vector<Row>> rows;                  // per scope, for the current object

  std::shared_ptr<const StringTable::Frozen> frozen;    // string ids as of the start of this flatten (lock-free lookups)
  std::map<std::string, VP> ns_private;                 // deep copy of the namespace cache
  const std::vector<std::string>* excluded = nullptr;   // excluder patterns of the calling process (may be empty)
  std::unordered_map<const Node*, VP> const_private;    // deep copies of constants captured by closures

  static VP deep_copy(const VP& v) {
    if (!v) return v;
    switch (v->t) {
      case VT::Null: return v_null();
      case VT::True: return v_bool(true);
      case VT::False: return v_bool(false);
      case VT::Num: return v_num(v->n);
      case VT::Str: return v_str(v->s);
      case VT::Arr:
      case VT::Set: {
        auto n = new_node();
        n->t = v->t;
        for (auto& x : v->items) n->items.push_back(deep_copy(x));
        return n;
      }
      default: {
        auto n = new_node();
        n->t = VT::Obj;
        for (auto& e : v->kv) n->kv.emplace_back(deep_copy(e.first), deep_copy(e.second));
        return n;
      }
    }
  }
  const VP& private_const(const VP& v) {
    auto it = const_private.find(v.get());
    if (it != const_private.end()) return it->second;
    return const_private.emplace(v.get(), deep_copy(v)).first->second;
  }

  VP data;   // {"inventory": ...}: what closures of referential templates read as `data`
  Flattener(Engine& e, const Compiled& cc, const std::map<std::string, VP>& ns_shared) : eng(e), c(cc) {
    if (cc.uses_data) data = e.data_doc();
    for (auto& kv : ns_shared) ns_private.emplace(kv.first, deep_copy(kv.second));
    rows.resize(c.schema.scopes.size());
    begin_chunk();
  }
  // the worker keeps its caches (evaluators, string ids, private namespace copies) across chunks; only the output resets
  void begin_chunk() {
    static_cast<ChunkOut&>(*this) = ChunkOut();
    ns_objs.clear();
    ns_row_of.clear();
    size_t ns = c.schema.scopes.size();
    hb.scope_off.resize(ns);
    for (size_t s = 1; s < ns; ++s) hb.scope_off[s].push_back(0);
    hb.scope_rows.assign(ns, 0);
    hb.cols.resize(c.schema.cols.size());
    for (size_t i = 0; i < hb.cols.size(); ++i)
      if (c.schema.cols[i].enc & GK_ENC_BYTES) hb.cols[i].boff.push_back(0);
    hb.name_off.push_back(0);
    hb.gen_off.push_back(0);
    hb.lbl_off.push_back(0);
    hb.nsn_off.push_back(0);
    hb.nsl_off.push_back(0);
  }
  std::unique_ptr<ChunkOut> take() { return std::unique_ptr<ChunkOut>(new ChunkOut(std::move(static_cast<ChunkOut&>(*this)))); }

  // Object data is only ever compared with constants the compiler interned, so values are LOOKED UP, never added:
  // an unknown string gets GK_SID_OTHER (equal to no constant).  The dictionary stays small and read-mostly.
  uint32_t sid(const std::string& key) {
    auto it = sid_cache.find(key);
    if (it != sid_cache.end()) return it->second;
    // the frozen copy answers without touching the table's lock (a reader lock is still an atomic update of one shared
    // cache line, 16 threads deep); only strings interned after the freeze need the locked path
    uint32_t id = GK_SID_UNDEF;
    auto fit = frozen->find(key);
    if (fit != frozen->end()) id = fit->second;
    else if (eng.strings().size_relaxed() != (uint32_t)frozen->size()) id = eng.strings().lookup(key);
    if (id == GK_SID_UNDEF) id = GK_SID_OTHER;
    if (sid_cache.size() > (1u << 18)) sid_cache.clear();
    sid_cache.emplace(key, id);
    return id;
  }
  // string values are by far the commonest: their cache is keyed by the raw string (no "s"-prefixed key is built on a hit)
  std::unordered_map<std::string, uint32_t> str_sid_cache;
  uint32_t sid_str(const std::string& raw) {
    auto it = str_sid_cache.find(raw);
    if (it != str_sid_cache.end()) return it->second;
    uint32_t id = sid("s" + raw);
    if (str_sid_cache.size() > (1u << 18)) str_sid_cache.clear();
    str_sid_cache.emplace(raw, id);
    return id;
  }
  uint32_t sid_value(const VP& v) { return v->t == VT::Str ? sid_str(v->s) : sid(intern_key(v)); }

  Eval& eval_for(const Closure& cl, const VP& input) {
    auto& slot = evals[cl.mod.get()];
    if (!slot) slot.reset(new Eval(*cl.mod, input, data));
    return *slot;
  }

  // Direct evaluation of a deterministic term.  `ok` is cleared when the term needs the general evaluator; a null result
  // with ok set means "undefined".
  VP eval_direct(const Term& t, const Env& env, const VP& input, Eval& ev, const Module& mod, bool& ok) {
    switch (t.k) {
      case TK::Scalar: return private_const(t.val);   // (never copy a literal of the shared AST: its reference count would bounce between workers)
      case TK::Var: {
        if (const VP* b = env.find(t.vid)) return *b;
        if (t.vid == mod.vid_input) return input;
        ok = false;
        return nullptr;
      }
      case TK::Ref: {
        VP cur = eval_direct(*t.head, env, input, ev, mod, ok);
        if (!ok || !cur) return nullptr;
        for (auto& a : t.args) {
          VP computed;
          if (a->k != TK::Scalar) computed = eval_direct(*a, env, input, ev, mod, ok);
          const VP& key = a->k == TK::Scalar ? a->val : computed;   // a literal key is only read: no copy, no reference-count traffic
          if (!ok) return nullptr;
          if (!key) return nullptr;
          if (cur->t == VT::Obj) cur = obj_get(cur, key);
          else if (cur->t == VT::Arr) {
            int64_t ix;
            if (key->t == VT::Num && num_fits_i64(key->n, &ix) && ix >= 0 && (size_t)ix < cur->items.size()) cur = cur->items[ix];
            else cur = nullptr;
          } else if (cur->t == VT::Set) cur = set_find(cur, key);
          else cur = nullptr;
          if (!cur) return nullptr;
        }
        return cur;
      }
      case TK::Call: {
        bool other_rule = false;
        const std::vector<Rule>* frules = ev.function_rules(t, &other_rule);
        const bool user = frules != nullptr;
        if (other_rule) {   // a non-function rule "called"
          ok = false;
          return nullptr;
        }
        if (user && t.args.size() != (*frules)[0].args.size()) {   // call with an output argument
          ok = false;
          return nullptr;
        }
        // argument vectors are recycled per nesting depth (a call inside a call's arguments uses the next one)
        if (call_depth_ >= arg_pool_.size()) arg_pool_.emplace_back();
        std::vector<VP>& args = arg_pool_[call_depth_];
        struct Depth {
          size_t& d;
          std::vector<VP>& v;
          Depth(size_t& x, std::vector<VP>& vv) : d(x), v(vv) { ++d; v.clear(); }
          ~Depth() { --d; v.clear(); }
        } guard(call_depth_, args);
        for (auto& a : t.args) {
          VP v = a->k == TK::Scalar ? private_const(a->val) : eval_direct(*a, env, input, ev, mod, ok);
          if (!ok) return nullptr;
          if (!v) return nullptr;   // an undefined argument makes the call undefined
          args.push_back(std::move(v));
        }
        if (user) return ev.call_function(*frules, args);
        bool known = true;
        VP v = call_builtin(t.name, args, &known);
        if (!known) ok = false;
        return v;
      }
      default: ok = false; return nullptr;
    }
  }

  // value of closure `cl` for the row `r` of scope cl.scope (chain resolved through parents)
  VP eval_closure(const Closure& cl, int scope, uint32_t r, const VP& input) {
    // move up to the closure's own scope
    while (scope != cl.scope && scope != 0) {
      r = rows[scope][r].parent;
      scope = c.schema.scopes[scope].parent;
    }
    if (cl.leaf == Closure::Elem) return rows[scope][r].elem;
    if (cl.leaf == Closure::Key) return rows[scope][r].key;
    // values of function calls and computed references are remembered for this object: the same closure feeds several
    // columns (a scope generator that is also a column; split(image, ":") under its count and under its last element)
    const Term& t = *cl.term;
    const bool memoise = t.k != TK::Ref || t.head->k != TK::Var || [&]() {
      for (auto& a : t.args)
        if (a->k != TK::Scalar) return true;
      return false;
    }();
    const uint64_t mkey = (uint64_t)(uintptr_t)&cl * 0x9E3779B97F4A7C15ull + r;
    if (memoise) {
      auto mit = memo.find(mkey);
      if (mit != memo.end()) return mit->second;
    }
    // environments are recycled per recursion depth (their storage is the only allocation a closure evaluation needs)
    if (env_depth >= env_pool.size()) env_pool.emplace_back();
    Env& env = env_pool[env_depth];
    env.b.clear();
    struct Depth {
      size_t& d;
      explicit Depth(size_t& x) : d(x) { ++d; }
      ~Depth() { --d; }
    } depth_guard(env_depth);
    for (auto& cap : cl.caps) {
      if (cap.second.k == CapArg::Conc) env.bind(cap.first, private_const(cap.second.v));
      else {
        const VP* v = eval_slot(*cap.second.col, scope, r, input);
        if (!v) return nullptr;
        env.bind(cap.first, *v);
      }
    }
    Eval& ev = eval_for(cl, input);
    // fast path: single-valued terms built from bound variables, constant paths and function calls are evaluated by a
    // direct recursion (no continuations, no environment growth); anything else -- iteration, comprehensions, rule
    // references -- goes through the general evaluator below
    {
      bool ok = true;
      VP v = eval_direct(t, env, input, ev, *cl.mod, ok);
      if (ok) {
        if (memoise) memo.emplace(mkey, v);
        return v;
      }
    }
    VP out = ev.eval_first(cl.term, env);
    if (memoise) memo.emplace(mkey, out);
    return out;
  }
  // ---- path closures: `<base>["a"]["b"][0]` with literal keys over `input`, a scope element or another closure -- most
  // columns.  They are walked in place: the result is a pointer to the value's slot inside its parent (no environment, no
  // evaluator, no reference-count traffic).  eval_slot() gives every other closure the same interface by parking its value
  // in `hold` until the object is done.
  struct PathPlan {
    bool is_path = false, from_input = false;
    const Closure* base = nullptr;
  };
  std::unordered_map<const Closure*, PathPlan> plans;
  const PathPlan& plan_of(const Closure& cl) {
    auto it = plans.find(&cl);
    if (it != plans.end()) return it->second;
    PathPlan pl;
    if (cl.leaf == Closure::None && cl.term->k == TK::Ref && cl.term->head->k == TK::Var) {
      bool lit = true;
      for (auto& a : cl.term->args) lit = lit && a->k == TK::Scalar;
      const int hv = cl.term->head->vid;
      const CapArg* cap = nullptr;
      for (auto& c2 : cl.caps)
        if (c2.first == hv) cap = &c2.second;
      if (lit && cap && cap->k == CapArg::Col) {
        pl.is_path = true;
        pl.base = cap->col.get();
      } else if (lit && !cap && hv == cl.mod->vid_input) {
        pl.is_path = pl.from_input = true;
      }
    }
    return plans.emplace(&cl, pl).first->second;
  }
  static const VP* child_slot(const Node& cur, const VP& key) {
    if (cur.t == VT::Obj) {
      size_t lo = 0, hi = cur.kv.size();
      const bool skey = key->t == VT::Str;
      while (lo < hi) {
        const size_t mid = (lo + hi) / 2;
        const VP& k = cur.kv[mid].first;
        const int c = (skey && k->t == VT::Str) ? k->s.compare(key->s) : v_cmp(k, key);
        if (c == 0) return &cur.kv[mid].second;
        if (c < 0) lo = mid + 1;
        else hi = mid;
      }
      return nullptr;
    }
    if (cur.t == VT::Arr) {
      int64_t ix;
      if (key->t == VT::Num && num_fits_i64(key->n, &ix) && ix >= 0 && (size_t)ix < cur.items.size()) return &cur.items[ix];
      return nullptr;
    }
    if (cur.t == VT::Set) {
      size_t lo = 0, hi = cur.items.size();
      while (lo < hi) {
        const size_t mid = (lo + hi) / 2;
        const int c = v_cmp(cur.items[mid], key);
        if (c == 0) return &cur.items[mid];
        if (c < 0) lo = mid + 1;
        else hi = mid;
      }
    }
    return nullptr;
  }
  std::deque<VP> hold;   // per object: values of non-path closures handed out by eval_slot (a deque never moves its elements)
  // slot of closure `cl`'s value for row `r` of `scope`, valid until the next object; nullptr = undefined
  const VP* eval_slot(const Closure& cl, int scope, uint32_t r, const VP& input) {
    if (cl.leaf != Closure::None) {
      while (scope != cl.scope && scope != 0) {
        r = rows[scope][r].parent;
        scope = c.schema.scopes[scope].parent;
      }
      const VP& v = cl.leaf == Closure::Elem ? rows[scope][r].elem : rows[scope][r].key;
      return v ? &v : nullptr;
    }
    const PathPlan& pl = plan_of(cl);
    if (pl.is_path) {
      const VP* cur = pl.from_input ? &input : eval_slot(*pl.base, scope, r, input);
      if (!cur || !*cur) return nullptr;
      for (auto& a : cl.term->args) {
        cur = child_slot(**cur, a->val);
        if (!cur) return nullptr;
      }
      return cur;
    }
    VP v = eval_closure(cl, scope, r, input);
    if (!v) return nullptr;
    hold.push_back(std::move(v));
    return &hold.back();
  }
  std::deque<std::vector<VP>> arg_pool_;
  size_t call_depth_ = 0;
  std::deque<Env> env_pool;   // (deque: a nested evaluation may grow it while outer references are live)
  size_t env_depth = 0;
  std::unordered_map<uint64_t, VP> memo;   // per object: (closure, row) -> value

  void header_row(const VP& o, const VP& ns, uint8_t source, bool present, bool second_row = false) {
    uint32_t fl = 0;
    uint32_t kind = GK_SID_UNDEF, group = GK_SID_UNDEF;
    uint64_t gvk = 0;
    if (present && o) {
      fl |= GK_F_HAS_OBJ;
      std::string g, v, k;
      split_gv(o, g, v, k);
      kind = sid_str(k);
      group = sid_str(g);
      if (!second_row) {   // (apiVersion, kind) of the object: is the batch of one kind?  (audit result order)
        uint64_t hh = 1469598103934665603ull;
        for (const std::string* part : {&g, &v, &k}) {
          for (unsigned char ch : *part) hh = (hh ^ ch) * 1099511628211ull;
          hh = (hh ^ 0xFFu) * 1099511628211ull;
        }
        hh |= 1ull;
        hb.gvk_lo = std::min(hb.gvk_lo, hh);
        hb.gvk_hi = std::max(hb.gvk_hi, hh);
        gvk = hh;
      }
      bool is_ns = k == "Namespace" && g.empty();
      if (is_ns) fl |= GK_F_IS_NS;
      std::string objns = meta_str(o, "namespace");
      if (!objns.empty()) fl |= GK_F_HAS_NS;
      if (ns) fl |= GK_F_NS_OBJ;
      std::string name = meta_str(o, "name"), gen = meta_str(o, "generateName");
      hb.name_bytes.insert(hb.name_bytes.end(), name.begin(), name.end());
      hb.gen_bytes.insert(hb.gen_bytes.end(), gen.begin(), gen.end());
      // name used by namespaces / excludedNamespaces -- match.go:118-179
      const std::string* nsn = nullptr;
      std::string nsmeta;
      if (is_ns) nsn = &name;
      else if (ns) nsmeta = meta_str(ns, "name"), nsn = &nsmeta;
      else if (!objns.empty()) nsn = &objns;
      if (nsn) {
        fl |= GK_F_NSNAME;
        hb.nsn_bytes.insert(hb.nsn_bytes.end(), nsn->begin(), nsn->end());
      }
      if (const Node* ls = labels_of(o))
        for (auto& e : ls->kv) {
          hb.lbl_kv.push_back(sid_str(e.first->s));
          hb.lbl_kv.push_back(sid_value(e.second));
        }
    }
    fl |= ((uint32_t)source << GK_F_SRC_SHIFT) & GK_F_SRC_MASK;
    if (!second_row) hb.gvk.push_back(gvk);
    hb.flags.push_back(fl);
    hb.kind_sid.push_back(kind);
    hb.group_sid.push_back(group);
    hb.nsn_off.push_back((uint32_t)hb.nsn_bytes.size());
    hb.name_off.push_back((uint32_t)hb.name_bytes.size());
    hb.gen_off.push_back((uint32_t)hb.gen_bytes.size());
    hb.lbl_off.push_back((uint32_t)hb.lbl_kv.size() / 2);
  }

  void encode(size_t ci, const VP& v) {
    const uint32_t enc = c.schema.cols[ci].enc;
    HostColumn& hc = hb.cols[ci];
    uint8_t vt = v ? (uint8_t)v->t : (uint8_t)GK_VT_UNDEF;
    int64_t num = 0;
    if (v && v->t == VT::Num && (enc & GK_ENC_NUM)) num = num_key(v->n);   // exact order against every integer constant (val.hpp)
    if (enc & GK_ENC_VT) hc.vt.push_back(vt);
    if (enc & GK_ENC_SID) hc.sid.push_back(v ? sid_value(v) : GK_SID_UNDEF);
    // non-numbers carry the extreme that OPA's cross-type order gives them relative to every number (null, booleans
    // below; strings, composites above): the device's ordered compares then need no type dispatch
    if (v && v->t != VT::Num && (enc & GK_ENC_NUM)) num = type_rank(v->t) < type_rank(VT::Num) ? INT64_MIN : INT64_MAX;
    if (enc & GK_ENC_NUM) hc.num.push_back(num);
    if (enc & GK_ENC_BYTES) {
      if (v && v->t == VT::Str) hc.bytes.insert(hc.bytes.end(), v->s.begin(), v->s.end());
      hc.boff.push_back((uint32_t)hc.bytes.size());
    }
    if (enc & GK_ENC_HEAD) {
      uint32_t h[GK_HEAD_WORDS] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (v && v->t == VT::Str) {
        size_t n = std::min<size_t>(v->s.size(), GK_HEAD_BYTES);
        memcpy(h, v->s.data(), n);
        reinterpret_cast<uint8_t*>(h)[GK_HEAD_WORDS * 4 - 1] = (uint8_t)std::min<size_t>(v->s.size(), 255);
      }
      hc.head.insert(hc.head.end(), h, h + GK_HEAD_WORDS);
    }
  }

  // placeholder rows for an object that is not evaluated (review error or excluded namespace): skipped by the kernel
  void placeholder() {
    const size_t nscopes = c.schema.scopes.size();
    size_t before = hb.flags.size();
    header_row(nullptr, nullptr, 0, false);
    hb.flags[before] |= GK_F_SKIP;
    std::swap(hb.flags, o_flags), std::swap(hb.kind_sid, o_kind), std::swap(hb.group_sid, o_group), std::swap(hb.nsn_off, o_nsn_off), std::swap(hb.nsn_bytes, o_nsn_bytes);
    std::swap(hb.name_off, o_name_off), std::swap(hb.gen_off, o_gen_off), std::swap(hb.lbl_off, o_lbl_off), std::swap(hb.lbl_kv, o_lbl_kv);
    std::swap(hb.name_bytes, o_name_bytes), std::swap(hb.gen_bytes, o_gen_bytes);
    header_row(nullptr, nullptr, 0, false, true);
    std::swap(hb.flags, o_flags), std::swap(hb.kind_sid, o_kind), std::swap(hb.group_sid, o_group), std::swap(hb.nsn_off, o_nsn_off), std::swap(hb.nsn_bytes, o_nsn_bytes);
    std::swap(hb.name_off, o_name_off), std::swap(hb.gen_off, o_gen_off), std::swap(hb.lbl_off, o_lbl_off), std::swap(hb.lbl_kv, o_lbl_kv);
    std::swap(hb.name_bytes, o_name_bytes), std::swap(hb.gen_bytes, o_gen_bytes);
    hb.nsrow.push_back(GK_NONE);
    for (size_t s = 1; s < nscopes; ++s) {
      // every parent row of this object gets an empty range; the root contributes exactly one row
      if (c.schema.scopes[s].parent == 0) hb.scope_off[s].push_back(hb.scope_off[s].back());
    }
    for (size_t ci = 0; ci < hb.cols.size(); ++ci)
      if (c.schema.cols[ci].scope == 0) encode(ci, nullptr);
    ++hb.n;
  }

  void add(const ObjIn& in) {
    std::string err;
    VP obj, old, ns;
    uint64_t tc0 = trace ? __builtin_ia32_rdtsc() : 0;
    VP doc = eng.review_doc(in, &obj, &old, &ns, &err, &ns_private);
    if (trace) doc_cycles += __builtin_ia32_rdtsc() - tc0;
    hb.obj_errors.push_back(err);
    const size_t nscopes = c.schema.scopes.size();
    if (!doc) return placeholder();
    // ---- stage 0: Excluder.IsNamespaceExcluded (excluder.go:95-127): a Namespace is tested by its own name, anything
    // else by its namespace (the webhook sets it from the request: pkg/webhook/common.go:181)
    if (excluded && !excluded->empty()) {
      const VP& ref = obj ? obj : old;
      std::string g, v, k;
      split_gv(ref, g, v, k);
      std::string subject = (k == "Namespace" && g.empty()) ? meta_str(ref, "name") : (in.ns_name ? std::string(in.ns_name) : meta_str(ref, "namespace"));
      bool skip = false;
      for (auto& p : *excluded) skip = skip || wildcard_match(p, subject);
      if (skip) doc = nullptr;   // falls into the placeholder path below: the kernel skips the row, no error text
    }
    if (!doc) return placeholder();
    // ---- header (object row, then old-object row into the side vectors)
    uint64_t th0 = trace ? __builtin_ia32_rdtsc() : 0;
    header_row(obj, ns, in.source, (bool)obj);
    std::swap(hb.flags, o_flags), std::swap(hb.kind_sid, o_kind), std::swap(hb.group_sid, o_group), std::swap(hb.nsn_off, o_nsn_off), std::swap(hb.nsn_bytes, o_nsn_bytes);
    std::swap(hb.name_off, o_name_off), std::swap(hb.gen_off, o_gen_off), std::swap(hb.lbl_off, o_lbl_off), std::swap(hb.lbl_kv, o_lbl_kv);
    std::swap(hb.name_bytes, o_name_bytes), std::swap(hb.gen_bytes, o_gen_bytes);
    bool old_distinct = old && old.get() != obj.get();
    header_row(old, ns, in.source, old_distinct, true);
    std::swap(hb.flags, o_flags), std::swap(hb.kind_sid, o_kind), std::swap(hb.group_sid, o_group), std::swap(hb.nsn_off, o_nsn_off), std::swap(hb.nsn_bytes, o_nsn_bytes);
    std::swap(hb.name_off, o_name_off), std::swap(hb.gen_off, o_gen_off), std::swap(hb.lbl_off, o_lbl_off), std::swap(hb.lbl_kv, o_lbl_kv);
    std::swap(hb.name_bytes, o_name_bytes), std::swap(hb.gen_bytes, o_gen_bytes);
    any_old = any_old || old_distinct;
    if (trace) hdr_cycles += __builtin_ia32_rdtsc() - th0;
    // ---- namespace table row
    if (ns) {
      auto it = ns_row_of.find(ns.get());
      uint32_t row;
      if (it == ns_row_of.end()) {
        row = (uint32_t)ns_objs.size();
        ns_objs.push_back(ns);
        ns_row_of.emplace(ns.get(), row);
        if (const Node* ls = labels_of(ns))
          for (auto& e : ls->kv) {
            hb.nsl_kv.push_back(sid_str(e.first->s));
            hb.nsl_kv.push_back(sid_value(e.second));
          }
        hb.nsl_off.push_back((uint32_t)hb.nsl_kv.size() / 2);
      } else {
        row = it->second;
      }
      hb.nsrow.push_back(row);
    } else {
      hb.nsrow.push_back(GK_NONE);
    }
    // ---- scopes + columns
    if (nscopes > 1 || !hb.cols.empty()) {
      VP input = v_obj({{v_str("review"), doc}});
      for (auto& e : evals) e.second->reset_input(input);
      memo.clear();
      hold.clear();
      for (auto& r : rows) r.clear();
      rows[0].push_back(Row{nullptr, nullptr, 0});
      for (size_t s = 1; s < nscopes; ++s) {
        const ScopeDef& sd = c.schema.scopes[s];
        auto& prow = rows[sd.parent];
        for (uint32_t pr = 0; pr < prow.size(); ++pr) {
          uint64_t t0 = trace ? __builtin_ia32_rdtsc() : 0;
          const VP* cslot = eval_slot(*sd.gen, sd.parent, pr, input);
          if (trace) scope_cycles[s] += __builtin_ia32_rdtsc() - t0;
          if (cslot) {
            const VP& coll = *cslot;
            if (coll->t == VT::Arr)
              for (size_t j = 0; j < coll->items.size(); ++j) rows[s].push_back(Row{coll->items[j], v_int((long long)j), pr});
            else if (coll->t == VT::Set)
              for (auto& x : coll->items) rows[s].push_back(Row{x, x, pr});
            else if (coll->t == VT::Obj)
              for (auto& e : coll->kv) rows[s].push_back(Row{e.second, e.first, pr});
          }
          hb.scope_off[s].push_back(hb.scope_rows[s] + (uint32_t)rows[s].size());
        }
      }
      for (size_t ci = 0; ci < hb.cols.size(); ++ci) {
        const ColDef& cd = c.schema.cols[ci];
        uint64_t t0 = trace ? __builtin_ia32_rdtsc() : 0;
        static const VP undefined;
        for (uint32_t r = 0; r < rows[cd.scope].size(); ++r) {
          const VP* v = eval_slot(*cd.expr, cd.scope, r, input);
          encode(ci, v ? *v : undefined);
        }
        if (trace) col_cycles[ci] += __builtin_ia32_rdtsc() - t0;
      }
      for (size_t s = 1; s < nscopes; ++s) hb.scope_rows[s] += (uint32_t)rows[s].size();
    }
    ++hb.n;
  }
  // ---- Lut closures of the device ingest path: the value for one tuple of leaf arguments.  The closure is evaluated by the
  // very code that flattens on the host (eval_slot), against skeleton documents that hold just the argument paths.
  struct Skel {
    VP val;                               // set: a leaf value
    std::map<std::string, Skel> obj;
    std::map<int64_t, Skel> arr;
    void put(const std::vector<VP>& keys, size_t i, const VP& v) {
      if (i == keys.size()) {
        val = v;
        return;
      }
      const VP& k = keys[i];
      int64_t ix;
      if (k->t == VT::Str) obj[k->s].put(keys, i + 1, v);
      else if (k->t == VT::Num && num_fits_i64(k->n, &ix) && ix >= 0 && ix < 4096) arr[ix].put(keys, i + 1, v);
    }
    VP build() const {
      if (val) return val;
      if (!arr.empty()) {
        std::vector<VP> items((size_t)arr.rbegin()->first + 1, v_null());
        for (auto& e : arr) items[(size_t)e.first] = e.second.build();
        return v_arr(std::move(items));
      }
      std::vector<std::pair<VP, VP>> kv;
      for (auto& e : obj) kv.emplace_back(v_str(e.first), e.second.build());
      return v_obj(std::move(kv));
    }
  };
  GkLutVal lut_value(const Closure& cl, const std::vector<XInfo::Arg>& args, const std::vector<VP>& vals) {
    Skel in_doc;
    std::map<int, Skel> elems;
    std::map<int, VP> keys;
    bool any_input = false;
    for (size_t a = 0; a < args.size(); ++a) {
      if (!vals[a]) continue;   // an undefined argument: its path is simply absent
      if (!args[a].leaf) {
        in_doc.put(args[a].keys, 0, vals[a]);
        any_input = true;
      } else if (args[a].leaf->leaf == Closure::Key) {
        if (args[a].keys.empty()) keys[args[a].leaf->scope] = vals[a];
      } else {
        elems[args[a].leaf->scope].put(args[a].keys, 0, vals[a]);
      }
    }
    VP input = any_input ? in_doc.build() : v_obj({{v_str("review"), v_obj({})}});
    for (auto& e : evals) e.second->reset_input(input);
    memo.clear();
    hold.clear();
    for (auto& r : rows) r.clear();
    rows[0].push_back(Row{nullptr, nullptr, 0});
    for (int sc = cl.scope; sc != 0; sc = c.schema.scopes[sc].parent) {
      Row r{nullptr, nullptr, 0};
      auto ei = elems.find(sc);
      if (ei != elems.end()) r.elem = ei->second.build();
      auto ki = keys.find(sc);
      if (ki != keys.end()) r.key = ki->second;
      rows[sc].push_back(r);
    }
    const VP* v = eval_slot(cl, cl.scope, 0, input);
    GkLutVal out;
    memset(&out, 0, sizeof out);
    out.vt = v ? (uint32_t)(*v)->t : (uint32_t)GK_VT_UNDEF;
    out.sid = v ? sid_value(*v) : GK_SID_UNDEF;
    if (v && (*v)->t == VT::Num) out.num = num_key((*v)->n);
    else if (v) out.num = type_rank((*v)->t) < type_rank(VT::Num) ? INT64_MIN : INT64_MAX;
    if (v && (*v)->t == VT::Str) {
      const std::string& str = (*v)->s;
      memcpy(out.head, str.data(), std::min<size_t>(str.size(), GK_HEAD_BYTES));
      reinterpret_cast<uint8_t*>(out.head)[GK_HEAD_WORDS * 4 - 1] = (uint8_t)std::min<size_t>(str.size(), 255);
    }
    return out;
  }
  bool trace = getenv("GK_FLATTEN_TRACE") != nullptr;
  std::vector<uint64_t> col_cycles = std::vector<uint64_t>(4096, 0), scope_cycles = std::vector<uint64_t>(256, 0);
  uint64_t doc_cycles = 0, hdr_cycles = 0, traced_objects = 0;
  ~Flattener() {
    if (!trace || traced_objects == 0) return;
    const uint64_t nobj = traced_objects;
    static std::mutex m;
    std::lock_guard<std::mutex> l(m);
    std::vector<std::pair<uint64_t, std::string>> v;
    for (size_t i = 0; i < c.schema.cols.size(); ++i) v.push_back({col_cycles[i], "col " + std::to_string(i) + " " + c.schema.cols[i].expr->key});
    for (size_t i = 1; i < c.schema.scopes.size(); ++i) v.push_back({scope_cycles[i], "scope " + std::to_string(i) + " " + c.schema.scopes[i].gen->key});
    v.push_back({doc_cycles, "review_doc (JSON parse)"});
    v.push_back({hdr_cycles, "header rows"});
    std::sort(v.rbegin(), v.rend());
    uint64_t tot = 0;
    for (auto& x : v) tot += x.first;
    fprintf(stderr, "[flatten worker] %llu objects, %.0f cycles/object accounted\n", (unsigned long long)nobj, (double)tot / nobj);
    for (size_t i = 0; i < v.size() && i < 25; ++i) fprintf(stderr, "  %7.0f cyc/obj  %.100s\n", (double)v[i].first / nobj, v[i].second.c_str());
  }
};

template <class T>
static void append(std::vector<T>& dst, const std::vector<T>& src) { dst.insert(dst.end(), src.begin(), src.end()); }
static void append_off(std::vector<uint32_t>& dst, const std::vector<uint32_t>& src, size_t skip_first) {
  uint32_t base = dst.empty() ? 0 : dst.back();
  for (size_t i = skip_first; i < src.size(); ++i) dst.push_back(base + src[i]);
}

void Engine::set_excluded_namespaces(const std::string& process, const std::vector<std::string>& patterns) {
  static const char* all[] = {"audit", "webhook", "mutation-webhook", "sync"};   // excluder.go:31-36 allProcesses
  std::unique_lock<std::shared_mutex> l(mu_);
  if (process == "*") {
    for (auto* p : all) excluded_[p] = patterns;
  } else {
    excluded_[process] = patterns;
  }
}
std::vector<std::string> Engine::excluded_namespaces(const std::string& process) {
  std::shared_lock<std::shared_mutex> l(mu_);
  auto it = excluded_.find(process);
  return it == excluded_.end() ? std::vector<std::string>() : it->second;
}

std::shared_ptr<HostBatch> Engine::flatten(const ObjIn* objs, size_t n, const Compiled& c, const std::string& process) {
  size_t T = std::min<size_t>((size_t)threads_, std::max<size_t>(1, n / 256));
  std::map<std::string, VP> ns_copy;
  std::vector<std::string> excluded;
  {
    std::shared_lock<std::shared_mutex> l(mu_);
    ns_copy = namespaces_;
    auto it = excluded_.find(process);
    if (!process.empty() && it != excluded_.end()) excluded = it->second;
  }
  auto frozen = strings_.freeze();
  // objects are handed out in chunks from a shared counter (threads on a throttled / shared host finish unevenly);
  // every chunk becomes one part, merged in object order below
  const size_t kChunk = T == 1 ? std::max<size_t>(n, 1) : 4096;
  const size_t nchunks = (n + kChunk - 1) / kChunk;
  std::vector<std::unique_ptr<ChunkOut>> parts(std::max<size_t>(nchunks, 1));
  std::vector<std::string> errs(T);
  std::atomic<size_t> next_chunk{0};
  auto work = [&](size_t t) {
    try {
      Flattener fl(*this, c, ns_copy);
      fl.excluded = &excluded;
      fl.frozen = frozen;
      for (;;) {
        const size_t k = next_chunk.fetch_add(1);
        if (k >= parts.size()) break;
        if (k) fl.begin_chunk();
        const size_t lo = k * kChunk, hi = std::min(n, lo + kChunk);
        for (size_t i = lo; i < hi; ++i) fl.add(objs[i]);
        fl.traced_objects += fl.hb.n;
        parts[k] = fl.take();
      }
    } catch (RegoError& e) {
      errs[t] = e.msg;
    } catch (std::exception& e) {
      errs[t] = e.what();
    }
  };
  auto tp0 = std::chrono::steady_clock::now();
  if (T == 1) work(0);
  else {
    std::vector<std::thread> th;
    for (size_t t = 0; t < T; ++t) th.emplace_back(work, t);
    for (auto& x : th) x.join();
  }
  auto tp1 = std::chrono::steady_clock::now();
  struct MergeTrace {
    std::chrono::steady_clock::time_point a, b;
    size_t T;
    ~MergeTrace() {
      if (getenv("GK_FLATTEN_TRACE"))
        fprintf(stderr, "[flatten] threads=%zu parallel part %.1f ms, merge %.1f ms\n", T, std::chrono::duration<double, std::milli>(b - a).count(),
                std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - b).count());
    }
  } trace{tp0, tp1, T};
  for (auto& e : errs)
    if (!e.empty()) throw RegoError{"flatten: " + e};
  // ---- merge
  auto out = std::make_shared<HostBatch>();
  HostBatch& hb = *out;
  hb.schema_version = c.version;
  const size_t nscopes = c.schema.scopes.size(), ncols = c.schema.cols.size();
  hb.scope_off.resize(nscopes);
  hb.scope_rows.assign(nscopes, 0);
  hb.cols.resize(ncols);
  hb.name_off.push_back(0);
  hb.gen_off.push_back(0);
  hb.lbl_off.push_back(0);
  hb.nsn_off.push_back(0);
  hb.nsl_off.push_back(0);
  for (size_t s = 1; s < nscopes; ++s) hb.scope_off[s].push_back(0);
  for (size_t i = 0; i < ncols; ++i)
    if (c.schema.cols[i].enc & GK_ENC_BYTES) hb.cols[i].boff.push_back(0);
  bool any_old = false;
  for (auto& p : parts) any_old = any_old || p->any_old;
  hb.has_old = any_old;
  // every destination array is one task (its parts are appended in order, into exactly-reserved storage); the tasks
  // run on all host threads -- the merge moves as many bytes as the H2D copy and must not be a serial tail
  std::vector<uint32_t> nsbase(parts.size(), 0);
  for (size_t pi = 0; pi < parts.size(); ++pi) {
    hb.n += parts[pi]->hb.n;
    if (pi + 1 < parts.size()) nsbase[pi + 1] = nsbase[pi] + (uint32_t)parts[pi]->hb.nsl_off.size() - 1;
    for (size_t s2 = 1; s2 < nscopes; ++s2) hb.scope_rows[s2] += parts[pi]->hb.scope_rows[s2];
  }
  std::vector<std::function<void()>> tasks;
  // plain concatenation of one member over all parts (then, with OldObject rows present, of its old-object twin)
#define GK_CAT(dst, member, oldmember)                                                   \
  tasks.push_back([&]() {                                                                \
    size_t tot = dst.size();                                                             \
    for (auto& p : parts) tot += p->hb.member.size() + (any_old ? p->oldmember.size() : 0); \
    dst.reserve(tot);                                                                    \
    for (auto& p : parts) append(dst, p->hb.member);                                     \
    if (any_old)                                                                         \
      for (auto& p : parts) append(dst, p->oldmember);                                   \
  })
#define GK_CAT_OFF(dst, member, oldmember)                                               \
  tasks.push_back([&]() {                                                                \
    size_t tot = dst.size();                                                             \
    for (auto& p : parts) tot += p->hb.member.size() + (any_old ? p->oldmember.size() : 0); \
    dst.reserve(tot);                                                                    \
    for (auto& p : parts) append_off(dst, p->hb.member, 1);                              \
    if (any_old)                                                                         \
      for (auto& p : parts) append_off(dst, p->oldmember, 1);                            \
  })
  GK_CAT(hb.flags, flags, o_flags);
  GK_CAT(hb.kind_sid, kind_sid, o_kind);
  GK_CAT(hb.group_sid, group_sid, o_group);
  GK_CAT_OFF(hb.name_off, name_off, o_name_off);
  GK_CAT_OFF(hb.gen_off, gen_off, o_gen_off);
  GK_CAT_OFF(hb.lbl_off, lbl_off, o_lbl_off);
  GK_CAT_OFF(hb.nsn_off, nsn_off, o_nsn_off);
  GK_CAT(hb.name_bytes, name_bytes, o_name_bytes);
  GK_CAT(hb.gen_bytes, gen_bytes, o_gen_bytes);
  GK_CAT(hb.nsn_bytes, nsn_bytes, o_nsn_bytes);
  GK_CAT(hb.lbl_kv, lbl_kv, o_lbl_kv);
#undef GK_CAT
#undef GK_CAT_OFF
  tasks.push_back([&]() {
    hb.nsrow.reserve(hb.n);
    for (size_t pi = 0; pi < parts.size(); ++pi)
      for (uint32_t r : parts[pi]->hb.nsrow) hb.nsrow.push_back(r == GK_NONE ? GK_NONE : r + nsbase[pi]);
  });
  tasks.push_back([&]() {
    for (auto& p : parts) append_off(hb.nsl_off, p->hb.nsl_off, 1);
  });
  tasks.push_back([&]() {
    for (auto& p : parts) append(hb.nsl_kv, p->hb.nsl_kv);
  });
  tasks.push_back([&]() {
    hb.obj_errors.reserve(hb.n);
    for (auto& p : parts) append(hb.obj_errors, p->hb.obj_errors);
    for (auto& p : parts) hb.gvk_lo = std::min(hb.gvk_lo, p->hb.gvk_lo), hb.gvk_hi = std::max(hb.gvk_hi, p->hb.gvk_hi);
  });
  tasks.push_back([&]() {
    hb.gvk.reserve(hb.n);
    for (auto& p : parts) append(hb.gvk, p->hb.gvk);
  });
  for (size_t s2 = 1; s2 < nscopes; ++s2)
    tasks.push_back([&, s2]() {
      size_t tot = 1;
      for (auto& p : parts) tot += p->hb.scope_off[s2].size();
      hb.scope_off[s2].reserve(tot);
      for (auto& p : parts) append_off(hb.scope_off[s2], p->hb.scope_off[s2], 1);
    });
  for (size_t i = 0; i < ncols; ++i) {
#define GK_COL(member)                                                  \
  tasks.push_back([&, i]() {                                            \
    size_t tot = 0;                                                     \
    for (auto& p : parts) tot += p->hb.cols[i].member.size();           \
    hb.cols[i].member.reserve(tot);                                     \
    for (auto& p : parts) append(hb.cols[i].member, p->hb.cols[i].member); \
  })
    GK_COL(vt);
    GK_COL(sid);
    GK_COL(num);
    GK_COL(bytes);
    GK_COL(head);
#undef GK_COL
    if (c.schema.cols[i].enc & GK_ENC_BYTES)
      tasks.push_back([&, i]() {
        for (auto& p : parts) append_off(hb.cols[i].boff, p->hb.cols[i].boff, 1);
      });
  }
  {
    const size_t MT = std::min<size_t>(std::max<size_t>(1, T), tasks.size());
    if (MT <= 1) {
      for (auto& t : tasks) t();
    } else {
      std::atomic<size_t> next{0};
      std::vector<std::thread> th;
      for (size_t t = 0; t < MT; ++t)
        th.emplace_back([&]() {
          for (;;) {
            size_t k = next.fetch_add(1);
            if (k >= tasks.size()) break;
            tasks[k]();
          }
        });
      for (auto& x : th) x.join();
    }
  }
  // ---- algorithmic bytes: every array the kernel may read, counted once
  uint64_t b = 0;
  auto sz = [&](auto& v) { b += (uint64_t)v.size() * sizeof(v[0]); };
  sz(hb.flags), sz(hb.kind_sid), sz(hb.group_sid), sz(hb.nsn_off), sz(hb.nsn_bytes), sz(hb.name_off), sz(hb.gen_off), sz(hb.lbl_off), sz(hb.lbl_kv);
  sz(hb.name_bytes), sz(hb.gen_bytes), sz(hb.nsrow), sz(hb.nsl_off), sz(hb.nsl_kv);
  for (size_t s = 1; s < nscopes; ++s) sz(hb.scope_off[s]);
  for (auto& col : hb.cols) sz(col.vt), sz(col.sid), sz(col.num), sz(col.boff), sz(col.bytes), sz(col.head);
  hb.alg_bytes = b;
  return out;
}

void Engine::add_expansion_template(const std::string& json) {
  std::unique_lock<std::shared_mutex> l(mu_);
  try {
    expansion_.upsert(json);
  } catch (std::runtime_error& e) {
    throw RegoError{e.what()};
  }
}
bool Engine::remove_expansion_template(const std::string& name) {
  std::unique_lock<std::shared_mutex> l(mu_);
  return expansion_.remove(name);
}
std::vector<std::string> Engine::expansion_conflicts() {
  std::shared_lock<std::shared_mutex> l(mu_);
  return expansion_.conflicts();
}
bool Engine::has_expansion() {
  std::shared_lock<std::shared_mutex> l(mu_);
  return !expansion_.empty();
}
uint64_t Engine::expansion_version() {
  std::shared_lock<std::shared_mutex> l(mu_);
  return expansion_.version();
}
bool Engine::expansion_selects(const std::string& g, const std::string& v, const std::string& k) {
  if (g.empty() && v.empty() && k.empty()) return true;   // (System.Expand: "cannot expand resource ... with empty GVK")
  std::shared_lock<std::shared_mutex> l(mu_);
  return expansion_.generates_from(g, v, k);
}
void Engine::expand_object(const ObjIn& in, std::vector<Resultant>& out) {
  // the generator is the request's object -- the OLD object of a DELETE (getReqObject, pkg/webhook/policy.go:435-440,599-603)
  const bool del = in.operation && std::string(in.operation) == "DELETE";
  const char* gj = del ? in.old_json : in.json;
  const size_t gl = del ? in.old_len : in.len;
  if (!gj) return;
  VP obj;
  try {
    obj = json_parse(gj, gl);
  } catch (JsonError&) {
    return;   // the review itself reports the undecodable object
  }
  if (!obj || obj->t != VT::Obj) return;
  if (in.ns_name) obj = ExpansionSystem::with_namespace(obj, in.ns_name);   // an admission request: obj.SetNamespace(req.Namespace) (policy.go:608)
  std::shared_lock<std::shared_mutex> l(mu_);
  // the review's Namespace object: the explicit one, else the cache entry for the request's namespace (policy.go:606-614)
  std::string nsn;
  bool have_ns = false;
  if (in.ns_json) {
    try {
      VP ns = json_parse(in.ns_json, in.ns_len);
      if (ns && ns->t == VT::Obj) nsn = meta_str(ns, "name"), have_ns = true;
    } catch (JsonError&) {
    }
  } else {
    const std::string key = in.ns_name ? std::string(in.ns_name) : meta_str(obj, "namespace");
    auto it = key.empty() ? namespaces_.end() : namespaces_.find(key);
    if (it != namespaces_.end()) nsn = meta_str(it->second, "name"), have_ns = true;
  }
  expansion_.expand(obj, have_ns ? &nsn : nullptr, out);
}

std::map<std::string, VP> Engine::namespaces_snapshot() {
  std::shared_lock<std::shared_mutex> l(mu_);
  std::map<std::string, VP> out;
  for (auto& kv : namespaces_) out.emplace(kv.first, v_deep_copy(kv.second));
  return out;
}

// ====================================================================================== device ingest: request + lookups
IngestReq Engine::ingest_request(const std::shared_ptr<const Compiled>& c, const uint8_t* blob, const unsigned long long* ooff, size_t n, uint32_t source,
                                 const std::string& process) {
  IngestReq rq;
  rq.blob = blob;
  rq.ooff = ooff;
  rq.n = n;
  rq.source = source;
  rq.c = c.get();
  rq.xprog = c->xprog;
  rq.strings = &strings_;
  {
    std::unique_lock<std::shared_mutex> l(mu_);
    auto it = excluded_.find(process);
    if (!process.empty() && it != excluded_.end()) rq.excluded = it->second;
    const uint32_t nstr = strings_.size();
    if (!ns_table_ || ns_table_version_ != ns_version_ || ns_table_strings_ != nstr) {
      // the namespace cache as device tables: label sids are looked up, never added (an unknown string equals no constant)
      auto t = std::make_shared<NsTableHost>();
      uint32_t cap = 64;
      while (cap < 4u * namespaces_.size()) cap <<= 1;
      t->tab.init(cap);
      auto sid_of = [&](const std::string& key) {
        const uint32_t id = strings_.lookup(key);
        return id == GK_SID_UNDEF ? (uint32_t)GK_SID_OTHER : id;
      };
      uint32_t row = 0;
      for (auto& kv : namespaces_) {
        t->tab.put(xhash(GK_SEED_NS, kv.first.data(), kv.first.size()), row++);
        if (const Node* ls = labels_of(kv.second))
          for (auto& e : ls->kv) {
            t->nsl_kv.push_back(sid_of("s" + e.first->s));
            t->nsl_kv.push_back(sid_of(intern_key(e.second)));
          }
        t->nsl_off.push_back((uint32_t)t->nsl_kv.size() / 2);
        const std::string nm = meta_str(kv.second, "name");
        t->nsn_bytes.insert(t->nsn_bytes.end(), nm.begin(), nm.end());
        t->nsn_off.push_back((uint32_t)t->nsn_bytes.size());
      }
      ns_table_ = t;
      ns_table_version_ = ns_version_;
      ns_table_strings_ = nstr;
    }
    rq.ns = ns_table_;
  }
  rq.lut_fill_from = [this, c](const uint8_t* b, const GkMiss* m, size_t k, std::vector<GkLutVal>& out) { lut_fill(*c, b, m, k, out); };
  rq.lut_fill = [this, c, blob](const GkMiss* m, size_t k, std::vector<GkLutVal>& out) { lut_fill(*c, blob, m, k, out); };
  return rq;
}

void Engine::lut_fill(const Compiled& c, const uint8_t* blob, const GkMiss* misses, size_t n, std::vector<GkLutVal>& out) {
  out.assign(n, GkLutVal{});
  if (!n) return;
  const XProgHost& xp = *c.xprog;
  std::map<std::string, VP> ns_copy;   // (Lut closures are pure: they never look at the namespace cache)
  auto frozen = strings_.freeze();
  const size_t T = std::min<size_t>((size_t)threads_, std::max<size_t>(1, n / 512));
  std::vector<std::string> errs(T);
  auto work = [&](size_t t) {
    try {
      Flattener fl(*this, c, ns_copy);
      fl.frozen = frozen;
      std::vector<VP> vals;
      for (size_t i = n * t / T; i < n * (t + 1) / T; ++i) {
        const GkMiss& m = misses[i];
        if (m.col == GK_CL_SIDVAL) {   // "the sid of this value": a number spelt non-canonically, a composite
          GkLutVal lv;
          memset(&lv, 0, sizeof lv);
          lv.sid = GK_SID_OTHER;
          if (m.args[0].kind == GK_ARG_JSON) {
            VP v = json_parse(reinterpret_cast<const char*>(blob) + m.args[0].off, m.args[0].len);
            lv.vt = (uint32_t)v->t;
            lv.sid = fl.sid_value(v);
          }
          out[i] = lv;
          continue;
        }
        if (m.col >= xp.cl.size() || !xp.cl_src[m.col]) throw RegoError{"device ingest: miss record names no lookup closure"};
        const auto& args = xp.cl_args[m.col];
        vals.assign(args.size(), nullptr);
        for (size_t a = 0; a < args.size() && a < GK_LUT_MAX_ARGS; ++a) {
          const GkMissArg& ma = m.args[a];
          switch (ma.kind) {
            case GK_ARG_JSON: vals[a] = json_parse(reinterpret_cast<const char*>(blob) + ma.off, ma.len); break;
            case GK_ARG_INDEX: vals[a] = v_int((long long)ma.off); break;
            case GK_ARG_SYNSTR: {   // a JSON string body: a slice of an escaped apiVersion keeps its escapes
              std::string s(ma.len ? reinterpret_cast<const char*>(blob) + ma.off : "", ma.len);
              vals[a] = s.find('\\') == std::string::npos ? v_str(std::move(s)) : json_parse(("\"" + s + "\"").data(), s.size() + 2);
              break;
            }
            default: break;
          }
        }
        out[i] = fl.lut_value(*xp.cl_src[m.col], args, vals);
      }
    } catch (RegoError& e) {
      errs[t] = e.msg;
    } catch (JsonError& e) {
      errs[t] = "device ingest: argument bytes do not parse: " + e.msg;
    } catch (std::exception& e) {
      errs[t] = e.what();
    }
  };
  if (T == 1) work(0);
  else {
    std::vector<std::thread> th;
    for (size_t t = 0; t < T; ++t) th.emplace_back(work, t);
    for (auto& x : th) x.join();
  }
  for (auto& e : errs)
    if (!e.empty()) throw RegoError{"lut_fill: " + e};
}

// ====================================================================================== materialisation
static std::string scoped_json(const std::vector<std::string>& v) {
  std::string o = "[";
  for (size_t i = 0; i < v.size(); ++i) {
    if (i) o += ",";
    json_quote(v[i], o);
  }
  return o + "]";
}

void Engine::materialize(const Compiled& c, const ObjIn& in, uint32_t obj_ix, uint32_t cix, const std::string& ep, std::vector<Violation>& out) {
  materialize_object(c, in, obj_ix, {Flagged{cix, false, 0}}, ep, out, nullptr);
}

void Engine::materialize_object(const Compiled& c, const ObjIn& in, uint32_t obj_ix, const std::vector<Flagged>& flagged,
                                const std::string& ep, std::vector<Violation>& out, VP* obj_out, MaterializeCtx* ctx) {
  MaterializeCtx local;
  if (!ctx) ctx = &local;
  ++ctx->epoch;
  std::string err;
  VP obj, old;
  VP doc = review_doc(in, &obj, &old, nullptr, &err);
  if (obj_out) *obj_out = obj ? obj : old;
  struct Rendered {
    std::vector<std::pair<std::string, std::string>> items;   // (msg, details JSON)
  };
  // constraints of one kind with equal parameters (e.g. the same policy scoped to different namespaces) render the same
  // messages for this object: evaluate once
  std::vector<std::pair<const Constraint*, Rendered>> memo;
  for (auto& f : flagged) {
    if (f.is_err) {
      autoreject(c, in, obj_ix, f.cix, f.err_code, ep, out);
      continue;
    }
    const Constraint& con = *c.order[f.cix];
    if (!doc) throw RegoError{"materialize: " + err};
    const Module& mod = *c.mods[f.cix];   // (pinned by the snapshot: no engine lock, no shared reference count per pair)
    size_t before = out.size();
    const std::string sc_json = scoped_json(con.action == "scoped" ? scoped_actions_for(con, ep) : std::vector<std::string>());
    const Rendered* rendered = nullptr;
    for (auto& m : memo)
      if (m.first->kind == con.kind && m.first->params_key == con.params_key) rendered = &m.second;
    if (!rendered) {
      memo.emplace_back(&con, Rendered());
      Rendered& r = memo.back().second;
      auto pit = ctx->params.find(&con);
      if (pit == ctx->params.end()) pit = ctx->params.emplace(&con, v_deep_copy(con.params)).first;
      VP inp = v_obj({{v_str("review"), doc}, {v_str("parameters"), pit->second}});
      // one evaluator per template and worker; within one object, switching constraints keeps the extents of
      // parameter-free helper rules (input_containers, ...)
      auto& slot = ctx->evals[&mod];
      uint64_t& seen = ctx->eval_epoch[&mod];
      if (c.uses_data && !ctx->data) ctx->data = data_doc();
      if (!slot) slot.reset(new Eval(mod, inp, ctx->data));
      else if (seen == ctx->epoch) slot->reset_parameters(inp);
      else slot->reset_input(inp);
      seen = ctx->epoch;
      Eval& ev = *slot;
      VP vs = ev.rule_value("violation");
      if (vs)
        for (auto& v : vs->items) {
          VP msg = obj_get(v, "msg");
          if (v->t != VT::Obj || !msg || msg->t != VT::Str) throw RegoError{"rego_type_error: violation element must be {\"msg\": string, ...}"};
          VP d = obj_get(v, "details");
          r.items.emplace_back(msg->s, d ? json_str(d) : "");
        }
      rendered = &r;
    }
    for (auto& it : rendered->items) {
      Violation x;
      x.object = obj_ix;
      x.constraint = f.cix;
      x.msg = it.first;
      x.details_json = it.second;
      x.action = con.action;
      x.scoped_json = sc_json;
      out.push_back(std::move(x));
    }
    if (out.size() == before)
      throw RegoError{"internal: GPU flagged (" + con.kind + "/" + con.name + ", object " + std::to_string(obj_ix) +
                      ") but the message renderer finds no violation -- lowering bug"};
  }
  // the evaluators keep the last input alive until their next reset: drop the document now (it is per object)
  for (auto& e : ctx->evals)
    if (ctx->eval_epoch[e.first] == ctx->epoch) e.second->reset_input(nullptr);
}

void Engine::autoreject(const Compiled& c, const ObjIn& in, uint32_t obj_ix, uint32_t cix, uint32_t code, const std::string& ep,
                        std::vector<Violation>& out) {
  const Constraint& con = *c.order[cix];
  std::string err;
  VP obj, old;
  (void)review_doc(in, &obj, &old, nullptr, &err);
  // matcher.go:58-60: the text names the object on which Matches failed -- Object first, OldObject if Object did not match
  VP ref = (code & GK_E_FROM_OLD) ? old : (obj ? obj : old);
  code &= GK_E_FROM_OLD - 1;
  std::string name = ref ? meta_str(ref, "name") : "";
  std::string detail;
  switch (code) {
    case GK_E_LSEL_INVALID: detail = c.match_errs[cix].lsel; break;
    case GK_E_NSSEL_INVALID: detail = c.match_errs[cix].nssel; break;
    case GK_E_NS_MISSING: detail = "namespace selector for namespace-scoped object but missing Namespace"; break;
    case GK_E_SRC_INVALID_MATCH: detail = c.match_errs[cix].src; break;
    case GK_E_SRC_UNSPECIFIED: detail = "source field not specified for resource " + name; break;
    case GK_E_SRC_INVALID_OBJ: detail = "invalid source field"; break;
    case GK_E_NUM_RANGE: detail = "number outside the exact int64 range in an ordered comparison"; break;
    default: break;
  }
  Violation x;
  x.object = obj_ix;
  x.constraint = cix;
  x.autoreject = true;
  // "unable to match constraints: <matcher error>": the frameworks client's wording of an autoreject (test/gator/test/test.bats:276)
  if (code == GK_E_NO_OBJECT) x.msg = "unable to match constraints: invalid request object: neither object nor old object are defined";
  else x.msg = "unable to match constraints: error matching the requested object: " + name + " :failed to run Match criteria: " + detail;   // matcher.go:58-60, match.go:52-54
  x.details_json = "{}";
  x.action = con.action;
  x.scoped_json = scoped_json(con.action == "scoped" ? scoped_actions_for(con, ep) : std::vector<std::string>());
  out.push_back(std::move(x));
}

}  // namespace gk
