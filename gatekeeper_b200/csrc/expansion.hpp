// Expansion of generator resources (a Deployment implies a Pod): the reference's pkg/expansion/system.go Expand + the
// aggregation rules of pkg/expansion/aggregate.go, run as a host pre-step of a review batch.  Callers in the reference:
// pkg/audit/manager.go:733-765 and pkg/webhook/policy.go:610-646.  Mutators are outside this engine's scope (the mutation
// system is not on the Client.Review path): resultants are reviewed as generated, unmutated.
#pragma once
#include <cstdint>
#include <map>
#include <string>
#include <vector>

#include "val.hpp"

namespace gk {

struct ExpansionTemplate {
  std::string name, source, action;     // spec.templateSource, spec.enforcementAction ("" = no override)
  std::string group, version, kind;     // spec.generatedGVK
  struct Apply {
    std::vector<std::string> groups, versions, kinds;
  };
  std::vector<Apply> apply;             // spec.applyTo
  bool applies_to(const std::string& g, const std::string& v, const std::string& k) const;
};

struct Resultant {
  VP obj;
  std::string template_name, action;
};

class ExpansionSystem {
 public:
  void upsert(const std::string& json);          // throws JsonError / std::runtime_error with ValidateTemplate's texts
  bool remove(const std::string& name);
  bool empty() const { return templates_.empty(); }
  // bumped by every upsert that stores a template (one that closes a cycle included) and every remove that removes one
  uint64_t version() const { return version_; }
  // some stored template, set aside or not, applies to (g, v, k): an object of that kind may have resultants
  bool generates_from(const std::string& g, const std::string& v, const std::string& k) const {
    for (auto& t : templates_)
      if (t.second.applies_to(g, v, k)) return true;
    return false;
  }
  std::vector<std::string> conflicts() const {   // System.GetConflicts -- system.go:81-83 (names, sorted)
    std::vector<std::string> out;
    for (auto& c : conflicted_)
      if (c.second) out.push_back(c.first);
    return out;
  }
  // System.Expand: every resultant of `obj`, grandchildren before children (system.go:137-167).  `ns_name`: the name of the
  // review's Namespace object, or null.  Throws std::runtime_error ("cannot expand resource ...", "could not find source field ...")
  void expand(const VP& obj, const std::string* ns_name, std::vector<Resultant>& out, int depth = 0) const;
  // aggregate.go:11,58-62
  // Unstructured.SetNamespace on a copy of `obj`: metadata.namespace = ns, or the field removed for ns == ""
  static VP with_namespace(const VP& obj, const std::string& ns);
  static std::string implied_by(const std::string& template_name, const std::string& msg) { return "[Implied by " + template_name + "] " + msg; }

 private:
  std::vector<const ExpansionTemplate*> templates_for(const std::string& g, const std::string& v, const std::string& k) const;
  void recompute_conflicts();
  std::map<std::string, ExpansionTemplate> templates_;
  uint64_t version_ = 0;
  std::map<std::string, bool> conflicted_;       // on a cycle of the generatedGVK -> applyTo graph: set aside (db.go hasConflicts)
};

VP expand_resource(const VP& obj, const std::string* ns_name, const ExpansionTemplate& t);   // expandResource -- system.go:203-247

}  // namespace gk
