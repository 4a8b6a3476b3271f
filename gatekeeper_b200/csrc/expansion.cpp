#include "expansion.hpp"

#include <algorithm>
#include <cctype>
#include <functional>
#include <set>
#include <stdexcept>

#include "engine.hpp"

namespace gk {

namespace {
std::string sf(const VP& o, const char* k) {
  VP v = obj_get(o, k);
  return v && v->t == VT::Str ? v->s : std::string();
}
std::vector<std::string> slist(const VP& o, const char* k) {
  std::vector<std::string> out;
  VP v = obj_get(o, k);
  if (v && v->t == VT::Arr)
    for (auto& x : v->items)
      if (x->t == VT::Str) out.push_back(x->s);
  return out;
}
bool has(const std::vector<std::string>& v, const std::string& s) { return std::find(v.begin(), v.end(), s) != v.end(); }
// a copy of object `o` with member `key` set
VP with(const VP& o, const std::string& key, VP val) {
  std::vector<std::pair<VP, VP>> kv;
  if (o && o->t == VT::Obj)
    for (auto& e : o->kv)
      if (e.first->s != key) kv.push_back(e);
  kv.emplace_back(v_str(key), std::move(val));
  return v_obj(std::move(kv));
}
}  // namespace

VP ExpansionSystem::with_namespace(const VP& obj, const std::string& ns) {
  VP md = obj_get(obj, "metadata");
  std::vector<std::pair<VP, VP>> kv;
  if (md && md->t == VT::Obj)
    for (auto& e : md->kv)
      if (e.first->s != "namespace") kv.push_back(e);
  if (!ns.empty()) kv.emplace_back(v_str("namespace"), v_str(ns));
  return with(obj, "metadata", v_obj(std::move(kv)));
}

bool ExpansionTemplate::applies_to(const std::string& g, const std::string& v, const std::string& k) const {
  for (auto& a : apply)   // ApplyTo.Matches -- pkg/mutation/match/apply_to.go:45-57
    if (has(a.groups, g) && has(a.versions, v) && has(a.kinds, k)) return true;
  return false;
}

void ExpansionSystem::upsert(const std::string& json) {
  VP t = json_parse(json.data(), json.size());
  ExpansionTemplate x;
  x.name = sf(obj_get(t, "metadata"), "name");
  VP spec = obj_get(t, "spec");
  x.source = sf(spec, "templateSource");
  x.action = sf(spec, "enforcementAction");
  VP gen = obj_get(spec, "generatedGVK");
  x.group = sf(gen, "group"), x.version = sf(gen, "version"), x.kind = sf(gen, "kind");
  VP ap = obj_get(spec, "applyTo");
  if (ap && ap->t == VT::Arr)
    for (auto& a : ap->items) x.apply.push_back({slist(a, "groups"), slist(a, "versions"), slist(a, "kinds")});
  // ValidateTemplate -- system.go:85-112
  if (x.name.empty()) throw std::runtime_error("ExpansionTemplate has empty name field");
  if (x.name.size() >= 64) throw std::runtime_error("ExpansionTemplate name must be less than 64 characters");
  if (x.source.empty()) throw std::runtime_error("ExpansionTemplate " + x.name + " has empty source field");
  if (x.group.empty() && x.version.empty() && x.kind.empty()) throw std::runtime_error("ExpansionTemplate " + x.name + " has empty generatedGVK field");
  if (x.apply.empty()) throw std::runtime_error("ExpansionTemplate " + x.name + " must specify ApplyTo");
  if (x.applies_to(x.group, x.version, x.kind))
    throw std::runtime_error("ExpansionTemplate " + x.name + " generates GVK " + x.group + "/" + x.version + ", Kind=" + x.kind + ", but also applies to that same GVK");
  const std::string name = x.name;
  templates_[name] = std::move(x);
  ++version_;
  recompute_conflicts();
  // db.upsert (db.go:222-245): the template is stored even when it closes a cycle -- it and the others on the cycle are set aside -- and the
  // caller is told (the reference's controller writes the error into the template's status)
  if (conflicted_[name]) throw std::runtime_error("template forms expansion cycle");
}

bool ExpansionSystem::remove(const std::string& name) {
  const bool had = templates_.erase(name) != 0;
  if (had) ++version_;
  recompute_conflicts();
  return had;
}

void ExpansionSystem::recompute_conflicts() {
  conflicted_.clear();
  // edge a -> b: a's generatedGVK matches b's applyTo; a template that can reach itself is on a cycle
  for (auto& a : templates_) {
    std::set<std::string> seen;
    std::vector<std::string> stack{a.first};
    bool cyc = false;
    while (!stack.empty() && !cyc) {
      const ExpansionTemplate& cur = templates_.at(stack.back());
      stack.pop_back();
      for (auto& b : templates_)
        if (b.second.applies_to(cur.group, cur.version, cur.kind)) {
          if (b.first == a.first) {
            cyc = true;
            break;
          }
          if (seen.insert(b.first).second) stack.push_back(b.first);
        }
    }
    conflicted_[a.first] = cyc;
  }
}

std::vector<const ExpansionTemplate*> ExpansionSystem::templates_for(const std::string& g, const std::string& v, const std::string& k) const {
  std::vector<const ExpansionTemplate*> out;
  for (auto& t : templates_) {   // (name order: the reference iterates a Go map, i.e. in no particular order)
    auto c = conflicted_.find(t.first);
    if (c != conflicted_.end() && c->second) continue;
    if (t.second.applies_to(g, v, k)) out.push_back(&t.second);
  }
  return out;
}

VP expand_resource(const VP& obj, const std::string* ns_name, const ExpansionTemplate& t) {
  if (t.source.empty()) throw std::runtime_error("cannot expand resource using a template with no source");
  if (t.group.empty() && t.version.empty() && t.kind.empty()) throw std::runtime_error("cannot expand resource using template with empty generatedGVK");
  const std::string pname = meta_str(obj, "name");
  VP cur = obj;
  size_t a = 0;
  while (a <= t.source.size()) {
    size_t b = t.source.find('.', a);
    if (b == std::string::npos) b = t.source.size();
    // unstructured.NestedMap (system.go:225-231): a missing key is "not found", walking into something that is not a map is an accessor error
    if (!cur || cur->t != VT::Obj) throw std::runtime_error("could not extract source field from unstructured");
    VP nx = obj_get(cur, t.source.substr(a, b - a).c_str());
    if (!nx) throw std::runtime_error("could not find source field \"" + t.source + "\" in resource " + pname);
    cur = nx;
    a = b + 1;
  }
  if (cur->t != VT::Obj) throw std::runtime_error("could not extract source field from unstructured");
  VP res = with(cur, "apiVersion", v_str(t.group.empty() ? t.version : t.group + "/" + t.version));
  res = with(res, "kind", v_str(t.kind));
  VP md = obj_get(res, "metadata");
  if (!md || md->t != VT::Obj) md = v_obj({});
  if (ns_name) {
    md = with(md, "namespace", v_str(*ns_name));
  } else {
    // unstructured.NestedString(obj, "metadata", "namespace") (system.go:239-246): absent is fine (a cluster-scoped parent), present but
    // not a string -- or a metadata that is not a map -- is an error
    VP pmd = obj_get(obj, "metadata");
    if (pmd && pmd->t != VT::Obj) throw std::runtime_error("could not extract namespace field \"" + t.source + "\" in parent resource " + pname);
    VP pns = pmd ? obj_get(pmd, "namespace") : nullptr;
    if (pns) {
      if (pns->t != VT::Str) throw std::runtime_error("could not extract namespace field \"" + t.source + "\" in parent resource " + pname);
      md = with(md, "namespace", pns);
    }
  }
  std::string mock = pname + (t.kind.empty() ? "" : "-") + t.kind;   // mockNameForResource -- system.go:289-297
  for (auto& ch : mock) ch = (char)std::tolower((unsigned char)ch);
  md = with(md, "name", v_str(mock));
  // ensureOwnerReference -- system.go:251-283
  const std::string pav = sf(obj, "apiVersion"), pk = sf(obj, "kind");
  if (!pav.empty() && !pk.empty() && !pname.empty()) {
    std::vector<VP> refs;
    VP old = obj_get(md, "ownerReferences");
    bool present = false;
    if (old && old->t == VT::Arr)
      for (auto& r : old->items) {
        refs.push_back(r);
        present = present || (sf(r, "apiVersion") == pav && sf(r, "kind") == pk && sf(r, "name") == pname);
      }
    if (!present) {
      refs.push_back(v_obj({{v_str("apiVersion"), v_str(pav)}, {v_str("kind"), v_str(pk)}, {v_str("name"), v_str(pname)}, {v_str("uid"), v_str("")}}));
      md = with(md, "ownerReferences", v_arr(std::move(refs)));
    }
  }
  return with(res, "metadata", md);
}

void ExpansionSystem::expand(const VP& obj, const std::string* ns_name, std::vector<Resultant>& out, int depth) const {
  if (depth >= 30) throw std::runtime_error("maximum recursion depth of 30 reached");   // maxRecursionDepth -- system.go:30
  std::string g, v, k;
  split_gv(obj, g, v, k);
  if (g.empty() && v.empty() && k.empty()) throw std::runtime_error("cannot expand resource " + meta_str(obj, "name") + " with empty GVK");
  std::vector<Resultant> res;
  for (auto* t : templates_for(g, v, k)) res.push_back(Resultant{expand_resource(obj, ns_name, *t), t->name, t->action});
  for (auto& r : res) expand(r.obj, ns_name, out, depth + 1);
  for (auto& r : res) out.push_back(std::move(r));
}

}  // namespace gk
