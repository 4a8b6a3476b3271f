"""Cases of the device ingest's edges, shared by the GPU tests (test_ingest_edges.py) and their host-emulation counterparts
(test_ingest_edges_hostemu.py): the review envelope of objects whose apiVersion, kind, name and namespace are spelt with JSON
escapes, the native string programs (split / trim / index / last / count over one leaf) at their edges against the lookup table's
answer for the same values, and pages with more distinct lookup arguments than the miss list and the table first hold.

Every case compares three results: the device ingest (ReviewBlob / upload_blob), the host flattener on the parsed documents
(ReviewBatch(..., materialize=False)) -- whole bitmaps and totals -- and the oracle's rendered results."""
import json
import random
import re

import numpy as np

from audit_order_cases import check_oracle, run_both, strip
from conftest import assert_same, engine_results, make_pair, oracle_results
from gatekeeper_b200 import driver as D
from gatekeeper_b200 import workloads as W
from oracle import audit as OA
from oracle import k8s


def _template(kind, body, helpers=""):
    return (kind, "package %s\n\nviolation[{\"msg\": msg}] {\n  %s\n}\n%s" % (kind.lower(), body, helpers))


def _con(kind, name, params=None, match=None):
    return W._constraint(kind, name, match=match, params=params)


def esc_char(ch):
    return "\\u%04x" % ord(ch)


def _page_parity(orc, drv, docs, ep=k8s.AUDIT_EP, flags=0, process="", drop=()):
    """ReviewBlob of the raw `docs` against the host flattener on the parsed documents (bitmaps and totals) and the oracle (results).
    Objects in `drop` (excluded by the process excluder) have no results.  Returns the device response."""
    dev = drv.ReviewBlob(W.PyBlob(docs), ep, flags=D.F_MATERIALIZE | flags)
    assert not any(dev.object_errors or []), [e for e in dev.object_errors if e][:3]
    objs = [json.loads(d) for d in docs]
    host = drv.ReviewBatch([D.Review(object=o, source="Original") for o in objs], ep, materialize=False, process=process)
    assert np.array_equal(np.asarray(host.viol_bits), np.asarray(dev.viol_bits)), "violation bitmap: the device ingest differs from the host flattener"
    assert np.array_equal(np.asarray(host.err_bits), np.asarray(dev.err_bits))
    assert list(host.totals) == list(dev.totals) and list(host.err_totals) == list(dev.err_totals)
    want = set()
    for i, o in enumerate(objs):
        if i in drop:
            continue
        want |= {(i,) + x[1:] for x in oracle_results(orc, [D.Review(object=o, source="Original")], ep)}
    assert_same(want, engine_results(dev))
    return dev


# ------------------------------------------------------------------------------------------------ the review envelope
ENV_TEMPLATES = [
    _template("K8sEnvGroup", 'input.review.kind.group == input.parameters.v\n  msg := sprintf("group %v", [input.review.kind.group])'),
    _template("K8sEnvVersion", 'input.review.kind.version == input.parameters.v\n  msg := sprintf("version %v", [input.review.kind.version])'),
    _template("K8sEnvKind", 'input.review.kind.kind == input.parameters.v\n  msg := sprintf("kind %v", [input.review.kind.kind])'),
    _template("K8sEnvName", 'input.review.name == input.parameters.v\n  msg := sprintf("name %v", [input.review.name])'),
    _template("K8sEnvNamespace", 'input.review.namespace == input.parameters.v\n  msg := sprintf("namespace %v", [input.review.namespace])'),
    # the group as a lookup argument (its bytes reach the host as a slice of the raw apiVersion)
    _template("K8sEnvGroupPrefix", 'startswith(input.review.kind.group, input.parameters.v)\n  msg := "group prefix"'),
    _template("K8sEnvAny", 'msg := sprintf("%v %v %v %v %v", [input.review.kind.group, input.review.kind.version, input.review.kind.kind, '
                           'input.review.name, input.review.namespace])'),
]
GROUPS = ["apps", "", "batch", "rbac.authorization.k8s.io"]
ENV_VALUES = {
    # the right answers, and the wrong ones a raw cut of an escaped apiVersion gives
    "K8sEnvGroup": GROUPS + ["apps\\", "app", "apps/v1"],
    "K8sEnvVersion": ["v1", "v1beta1", "apps/v1", "/v1", "v", "1"],
    "K8sEnvKind": ["Deployment", "Pod", "Namespace", "Job", "ClusterRole"],
    "K8sEnvName": ["web", "a.b-c", "prod", "kube-system", "x"],
    "K8sEnvNamespace": ["prod", "kube-system", "default", "team-a"],
    "K8sEnvGroupPrefix": ["app", "apps", "rbac.", ""],
}
ENV_MATCH = {
    "apps-deploy": {"kinds": [{"apiGroups": ["apps"], "kinds": ["Deployment"]}]},
    "core": {"kinds": [{"apiGroups": [""], "kinds": ["*"]}]},
    "core-ns": {"kinds": [{"apiGroups": [""], "kinds": ["Namespace"]}]},
    "batch-any": {"kinds": [{"apiGroups": ["batch", "rbac.authorization.k8s.io"], "kinds": ["*"]}]},
    "prod": {"namespaces": ["prod"]},
    "not-kube": {"excludedNamespaces": ["kube-*"]},
    "cluster": {"scope": "Cluster"},
    "namespaced": {"scope": "Namespaced"},
}
GVKS = [("apps/v1", "Deployment"), ("v1", "Pod"), ("batch/v1", "Job"), ("v1", "Namespace"), ("rbac.authorization.k8s.io/v1", "ClusterRole"),
        ("apps/v1beta1", "Deployment")]
CLUSTER_SCOPED = ("Namespace", "ClusterRole")


def spell(s, how):
    """`s` as the body of a JSON string: raw, '/' as "\\/" or as a \\u escape, one letter (first, middle, last) or every character
    as a \\u escape."""
    if how == "raw" or not s:
        return s
    if how == "slash":
        return s.replace("/", "\\/")
    if how == "u2f":
        return s.replace("/", "\\u002f")
    if how == "U2F":
        return s.replace("/", "\\u002F")
    if how == "whole":
        return "".join(esc_char(ch) for ch in s)
    at = {"first": 0, "mid": len(s) // 2, "last": len(s) - 1}[how]
    return s[:at] + esc_char(s[at]) + s[at + 1:]


SPELLINGS = ("raw", "slash", "u2f", "U2F", "first", "mid", "last", "whole")


def envelope_doc(api, kind, name, ns, sp_api, sp_kind, sp_name, sp_ns, extra=""):
    meta = '"name":"%s"' % spell(name, sp_name)
    if ns is not None:
        meta += ',"namespace":"%s"' % spell(ns, sp_ns)
    return ('{"apiVersion":"%s","kind":"%s","metadata":{%s}%s}' % (spell(api, sp_api), spell(kind, sp_kind), meta, extra)).encode()


def envelope_docs(seed=11):
    """Every GVK with its apiVersion in every spelling; kind, name and namespace in a rotating spelling of their own."""
    rnd = random.Random(seed)
    docs = []
    for gi, (api, kind) in enumerate(GVKS):
        for si, sp in enumerate(SPELLINGS):
            for j in range(3):
                name = ("web", "a.b-c", "x", "prod", "kube-system")[(si + j) % 5] if kind != "Namespace" else ("prod", "kube-system", "team-a")[j]
                ns = None if kind in CLUSTER_SCOPED else ("prod", "kube-system", "default", "team-a")[(gi + si + j) % 4]
                docs.append(envelope_doc(api, kind, name, ns, sp, SPELLINGS[(si + j + 1) % 8], SPELLINGS[(si + 2 * j) % 8],
                                         SPELLINGS[(si + j + 3) % 8]))
    # the Namespace kind with an escaped letter in its middle, a core version written as escapes, a Deployment with a body
    docs.append(b'{"apiVersion":"v1","kind":"Name\\u0073pace","metadata":{"name":"kube-public"}}')
    docs.append(b'{"apiVersion":"v\\u0031","kind":"Namespace","metadata":{"name":"prod"}}')
    docs.append(b'{"apiVersion":"apps\\/v1","kind":"Deployment","metadata":{"name":"web","namespace":"prod"},"spec":{"replicas":1}}')
    # escapes that decode to more than one byte, and a surrogate pair, in the group
    docs.append('{"apiVersion":"gr\\u00fcn.example\\/v1","kind":"Pod","metadata":{"name":"web","namespace":"prod"}}'.encode())
    docs.append('{"apiVersion":"\\ud83d\\ude00.example\\u002fv2","kind":"Pod","metadata":{"name":"web","namespace":"prod"}}'.encode())
    # a '/' only in the version part after an escaped one, and no '/' at all but escapes
    docs.append(b'{"apiVersion":"a\\/b/c","kind":"Pod","metadata":{"name":"web","namespace":"prod"}}')
    docs.append(b'{"apiVersion":"\\u0076\\u0031","kind":"Pod","metadata":{"name":"web","namespace":"prod"}}')
    rnd.shuffle(docs)
    return docs


def envelope_engine(lib):
    cons = [_con(k, "%s-%d" % (k.lower(), i), params={"v": v}) for k, vals in ENV_VALUES.items() for i, v in enumerate(vals)]
    cons += [_con("K8sEnvAny", name, match=m) for name, m in ENV_MATCH.items()]
    nss = [{"apiVersion": "v1", "kind": "Namespace", "metadata": {"name": n, "labels": {"env": n}}} for n in ("prod", "default")]
    orc, drv, _ = make_pair(ENV_TEMPLATES, cons, nss, lib_path=lib)
    assert "ingest: device" in drv.Dump(), drv.Dump().splitlines()[:3]
    return orc, drv, nss


def case_envelope(lib, excluded=("kube-*",)):
    """Objects whose apiVersion, kind, name and namespace are spelt with escapes (\\/, \\u002f as the group separator, \\u00XX for a
    letter, first, last or everywhere): the device ingest, the host flattener and the oracle agree on every template that reads the
    envelope and on every match by apiGroups / kinds / namespaces / excludedNamespaces / scope.  Then under the audit process's
    excluder, and through the ordered audit on a page of one GVK in mixed spellings, which must be classified as one kind."""
    orc, drv, nss = envelope_engine(lib)
    docs = envelope_docs()
    dev = _page_parity(orc, drv, docs)
    assert sum(dev.totals) > len(docs)
    # the process excluder: a Namespace by its own name (kind spelt with escapes included), anything else by its namespace
    drv.SetExcludedNamespaces("audit", list(excluded))
    objs = [json.loads(d) for d in docs]
    drop = {i for i, o in enumerate(objs) if k8s.is_namespace_excluded(excluded, o)}
    assert drop and any(o["kind"] == "Namespace" for i, o in enumerate(objs) if i in drop)
    _page_parity(orc, drv, docs, flags=D.PROCESS_FLAG["audit"], process="audit", drop=drop)
    # the ordered audit: the whole mixed page, then a page of one GVK in every spelling (one kind: the lazy path)
    nsmap = {x["metadata"]["name"]: x for x in nss}
    one = [envelope_doc("apps/v1", "Deployment", "d-%02d" % i, ("prod", "default")[i % 2], SPELLINGS[i % 8], SPELLINGS[(i // 8) % 8], "raw", "raw")
           for i in range(40)]
    for page, limit in ((docs, 5), (one, 3)):
        pb = W.PyBlob(page)
        po = [json.loads(d) for d in page]
        dev_rb = drv.upload_blob(pb, process="audit")
        host_rb = drv.upload([D.Review(object=o, source="Original") for o in po], process="audit")
        d_plain, d_ordered = run_both(drv, [(pb, dev_rb)], limit)
        h_plain, h_ordered = run_both(drv, [(None, host_rb)], limit)
        assert d_plain == h_plain and d_ordered == h_ordered
        assert strip(d_plain) == strip(d_ordered)
        check_oracle(d_ordered, OA.audit(orc, po, namespaces=nsmap, excluded_namespaces=excluded, limit=limit))
        if page is one:
            assert d_plain["pairsCounted"] > 0, "a page of one GVK in several spellings was not classified as one kind"
        dev_rb.free()
        host_rb.free()
    drv.close()
    return len(docs)


# ------------------------------------------------------------------------------------------------ native string programs
SX_HELPERS = {
    "K8sSxIndex": ('f(x) = t { parts := split(x, ":"); t := parts[1] }', str),
    "K8sSxIndexPast": ('f(x) = t { parts := split(x, ":"); t := parts[3] }', str),
    "K8sSxOverlap0": ('f(x) = t { parts := split(x, "aa"); t := parts[0] }', str),
    "K8sSxOverlap2": ('f(x) = t { parts := split(x, "aa"); t := parts[2] }', str),
    "K8sSxLast": ('f(x) = t { parts := split(x, "/"); t := parts[count(parts) - 1] }', str),
    "K8sSxCount": ('f(x) = n { n := count(split(x, ",")) }', int),
    "K8sSxTrim": ('f(x) = t { t := trim(x, "-.") }', str),
    "K8sSxTrimCount": ('f(x) = n { n := count(trim(x, "-")) }', int),
    # (a split of a split's segment is not compiled to a native program: the lookup table answers it for every row)
    "K8sSxNested": ('f(x) = t { a := split(x, "@"); b := split(a[0], ":"); t := b[1] }', str),
}
SX_NATIVE = [k for k in SX_HELPERS if k != "K8sSxNested"]


def sx_want(kind, s):
    """The helper's value for the string `s` (Go's strings.Split / strings.Trim, counts in code points), or None when undefined."""
    def at(parts, i):
        return parts[i] if 0 <= i < len(parts) else None
    return {"K8sSxIndex": lambda: at(s.split(":"), 1), "K8sSxIndexPast": lambda: at(s.split(":"), 3),
            "K8sSxOverlap0": lambda: at(s.split("aa"), 0), "K8sSxOverlap2": lambda: at(s.split("aa"), 2),
            "K8sSxLast": lambda: s.split("/")[-1], "K8sSxCount": lambda: len(s.split(",")),
            "K8sSxTrim": lambda: s.strip("-."), "K8sSxTrimCount": lambda: len(s.strip("-")),
            "K8sSxNested": lambda: at(s.split("@")[0].split(":"), 1)}[kind]()


# every edge of the programs: empty, only delimiters, leading / trailing / doubled delimiters, a delimiter that overlaps itself, an
# index past the last segment, no delimiter at all, a cutset that trims everything, nested splits -- at 0, 1, 2, ~8 and ~16 bytes
SX_VALUES = ["", ":", "a", "/", ",", "-", "@", "::", "a:", ":a", "ab", "aa", "//", ",,", "--", "-.", "@:",
             "aaa", "aaaa", "aaaaa", "a:b", "a/b", "a,b", ".a.", "x@y", ":::::::", "a:b:c:d", "aaaaaaaa", "abcdefgh", "-.-.-.-.",
             "abc/def/", "/abcdefg", "x@a:b@c", "u:v@w:x", "a,,b,c,", "--a-b--.", "abcdefghijklmnop", "aaaaaaaaaaaaaaaa",
             "::::::::::::::::", "a:bcdefghijklmn:", "/a/b/c/d/e/f/g/h", "img:v1.2@sha:abc", "-.-.-.-.-.-.-.-.", ",a,b,c,d,e,f,g,h",
             "aabaabaabaabaaba", "..............x."]
SX_NON_ASCII = ["\u00e9:\u00fc", "a:\u00f6", "\u2603/x", "\u00fc", "-\u00e9-", "a\u00e9aa:b"]
SX_NON_STRING = ["5", "null", "true", '{"a":":"}', '[":"]', "1.5", None]   # (JSON text of the leaf; None: the key is absent)


def sx_doc(i, leaf_json):
    ann = '"annotations":{"s":%s},' % leaf_json if leaf_json is not None else ""
    return ('{"apiVersion":"v1","kind":"ConfigMap","metadata":{%s"name":"o-%03d","namespace":"default"}}' % (ann, i)).encode()


def sx_escaped(s, k):
    """JSON text of `s` with its character at k % len written as a \\u00XX escape."""
    at = k % len(s)
    return '"%s"' % (s[:at] + esc_char(s[at]) + s[at + 1:])


def sx_engine(lib, kinds=tuple(SX_HELPERS)):
    tm, cons = [], []
    for kind in kinds:
        helper, typ = SX_HELPERS[kind]
        field = "n" if typ is int else "v"
        tm.append(_template(kind, 'y := f(input.review.object.metadata.annotations.s)\n  y == input.parameters.%s\n  msg := sprintf("%%v", [y])' % field,
                            helper + "\n"))
        outs = sorted({sx_want(kind, s) for s in SX_VALUES + SX_NON_ASCII} - {None}, key=repr)
        cons += [_con(kind, "%s-%d" % (kind.lower(), j), params={field: v}) for j, v in enumerate(outs)]
    orc, drv, _ = make_pair(tm, cons, lib_path=lib)
    assert "ingest: device" in drv.Dump(), drv.Dump().splitlines()[:3]
    return orc, drv, cons


TRACE_MISSES = re.compile(r"lookups missed \(host-evaluated\) (\d+)|lookups: (\d+) missed")


def traced_misses(capfd, run):
    """Run `run` with GK_TRACE_INGEST=1 set by the caller; the lookups the ingest sent to the host, from its trace line on stderr."""
    capfd.readouterr()
    run()
    err = capfd.readouterr().err
    hits = TRACE_MISSES.findall(err)
    assert len(hits) == 1, err[-2000:]
    return int(hits[0][0] or hits[0][1])


def case_string_programs(lib, monkeypatch, capfd):
    """Every GK_SX_* shape over every edge value, raw (the native program runs) and with one character escaped (the lookup table
    answers): their bitmap rows are equal, equal to the host flattener's and to the oracle's.  The ingest trace proves the path: no
    lookup for the raw ASCII page, lookups for the escaped one.  Non-ASCII and non-string leaves go through the table too."""
    monkeypatch.setenv("GK_TRACE_INGEST", "1")
    raw = [sx_doc(i, '"%s"' % s) for i, s in enumerate(SX_VALUES)]
    escd = [sx_doc(i, sx_escaped(s, i)) for i, s in enumerate(SX_VALUES) if s]
    other = [sx_doc(900 + i, json.dumps(s)) for i, s in enumerate(SX_NON_ASCII)] + [sx_doc(950 + i, s) for i, s in enumerate(SX_NON_STRING)]
    other += [sx_doc(980 + i, json.dumps(s, ensure_ascii=False)) for i, s in enumerate(SX_NON_ASCII)]   # (raw UTF-8 bytes)
    for page, native in ((raw, True), (escd, False)):
        orc, drv, _ = sx_engine(lib, SX_NATIVE)
        n = traced_misses(capfd, lambda: drv.ReviewBlob(W.PyBlob(page), k8s.AUDIT_EP, with_results=False))
        assert (n == 0) if native else (n > 0), (native, n)
        drv.close()
    orc, drv, cons = sx_engine(lib)
    docs = raw + escd + other
    dev = _page_parity(orc, drv, docs)
    bits = np.asarray(dev.viol_bits)
    nonempty = [i for i, s in enumerate(SX_VALUES) if s]
    for j, i in enumerate(nonempty):
        assert np.array_equal(bits[i], bits[len(raw) + j]), (SX_VALUES[i], "the lookup table's answer differs from the native program's")
    # every object of the raw page violates the constraints of the helpers it defines: one per defined helper
    assert sum(dev.totals) >= sum(1 for s in SX_VALUES for k in SX_HELPERS if sx_want(k, s) is not None)
    drv.close()
    return int(sum(dev.totals))


# ------------------------------------------------------------------------------------------------ many distinct lookup arguments
CPU_SPELLINGS = ('"%dm"', '"0.%06d"', '%d', '"%d"')         # (JSON text; plain integers only: another number spelling adds a lookup)
MEM_SPELLINGS = ('"%dMi"', '"%dGi"', '%d', '"%dKi"')


LOOKUPS_PER_LIMIT = 2   # lookup closures of K8sContainerLimits over one limit (canonify_cpu / canonify_mem, and the test of it)


def limits_pods(n, start=0, per_pod=8, repeat_every=10):
    """`n` Pods of `per_pod` containers, each with its own limits.cpu and limits.memory in a rotating spelling; every
    `repeat_every`-th Pod repeats the previous one's limits, so that some arguments recur.  Returns the documents and the set of
    distinct (field, JSON text) arguments."""
    docs, args = [], set()
    for i in range(start, start + n):
        src = i - 1 if i % repeat_every == repeat_every - 1 else i
        cs = []
        for j in range(per_pod):
            k = src * per_pod + j
            cpu, mem = CPU_SPELLINGS[k % 4] % k, MEM_SPELLINGS[(k // 4) % 4] % k
            args.add(("cpu", cpu))
            args.add(("mem", mem))
            cs.append('{"name":"c%d","image":"gcr.io/a:v1","resources":{"limits":{"cpu":%s,"memory":%s}}}' % (j, cpu, mem))
        docs.append(('{"apiVersion":"v1","kind":"Pod","metadata":{"name":"p-%06d","namespace":"default"},"spec":{"containers":[%s]}}'
                     % (i, ",".join(cs))).encode())
    return docs, args


def limits_engine(lib, with_constraints=True):
    t = W.templates()["containerlimits"]
    cons = [_con(t["kind"], "limits-%d" % i, params=p) for i, p in enumerate(W.CONFIG2_PARAMS["containerlimits"])]
    orc, drv, _ = make_pair([(t["kind"], t["rego"])], cons if with_constraints else [], lib_path=lib)
    return orc, drv, cons


def _bits(resp):
    return np.array(resp.viol_bits, copy=True), np.array(resp.err_bits, copy=True), list(resp.totals), list(resp.err_totals)


def _same_bits(a, b, what):
    for x, y, part in zip(a, b, ("violation bitmap", "error bitmap", "totals", "error totals")):
        assert np.array_equal(np.asarray(x), np.asarray(y)), "%s: %s differs" % (what, part)


def case_many_lookups(lib, monkeypatch, capfd, n, sample=300, n_patch=0, n_drop=0):
    """`n` Pods whose containers' limits are (nearly all) distinct lookup arguments of K8sContainerLimits' canonify_cpu /
    canonify_mem: more than one round's miss list holds, and enough to grow the lookup table inside one upload.  The device
    bitmap and totals equal the host flattener's on the whole page, the oracle's on a sample that holds the last object, and the
    ingest trace counts exactly one lookup per distinct argument -- none lost to the full miss list or dropped by the growth.
    With `n_patch`: the same page kept on the device and refreshed after the constraints arrive, then patched (`n_drop` objects
    dropped, `n_patch` new ones appended), each equal to a fresh upload of the resulting page."""
    monkeypatch.setenv("GK_TRACE_INGEST", "1")
    # the chosen spellings start no lookup but the template's: a small page counts LOOKUPS_PER_LIMIT per distinct argument
    small, small_args = limits_pods(40, start=10 ** 6)
    orc, drv, _ = limits_engine(lib)
    assert "ingest: device" in drv.Dump(), drv.Dump().splitlines()[:3]
    assert traced_misses(capfd, lambda: drv.ReviewBlob(W.PyBlob(small), k8s.AUDIT_EP, with_results=False)) == LOOKUPS_PER_LIMIT * len(small_args)
    drv.close()
    docs, args = limits_pods(n)
    page = W.PyBlob(docs)
    orc, drv, cons = limits_engine(lib)
    holder = {}
    misses = traced_misses(capfd, lambda: holder.setdefault("rb", drv.upload_blob(page)))
    rb = holder["rb"]
    assert misses == LOOKUPS_PER_LIMIT * len(args), (misses, len(args))
    dev = rb.eval(k8s.AUDIT_EP)
    got = _bits(dev)
    host = drv.ReviewBatch([D.Review(object=json.loads(d), source="Original") for d in docs], k8s.AUDIT_EP, materialize=False)
    _same_bits(_bits(host), got, "the device ingest against the host flattener")
    assert sum(got[2]) > 0
    objs = sorted(set(random.Random(n).sample(range(n), min(n, sample - 1))) | {n - 1})
    want = set()
    for o in objs:
        want |= {(o, x[1]) for x in oracle_results(orc, [D.Review(object=json.loads(docs[o]), source="Original")], k8s.AUDIT_EP)}
    keys = list(dev.constraints)
    have = {(o, keys[c]) for o in objs for c in range(len(keys)) if (int(got[0][o, c // 32]) >> (c % 32)) & 1}
    assert_same(want, have)
    rb.free()
    drv.close()
    if not n_patch:
        return misses
    # refresh: kept on the device without the constraints, re-extracted (lookups from the device copy) once they arrive
    _, drv, _ = limits_engine(lib, with_constraints=False)
    rb = drv.upload_blob(page, keep_source=True)
    for c in cons:
        drv.AddConstraint(c)
    assert rb.refresh()["rebuilt"]
    _same_bits(_bits(rb.eval(k8s.AUDIT_EP)), got, "refresh against a fresh upload")
    # patch: drop some objects, append new ones with values of their own
    drop = sorted(random.Random(7).sample(range(n), n_drop))
    add, _ = limits_pods(n_patch, start=2 * n)
    assert rb.patch(drop, add)["n"] == n - n_drop + n_patch
    patched = _bits(rb.eval(k8s.AUDIT_EP))
    dropped = set(drop)
    result = [d for i, d in enumerate(docs) if i not in dropped] + add
    rb.free()
    drv.close()
    _, drv, _ = limits_engine(lib)
    fresh = drv.upload_blob(W.PyBlob(result))
    _same_bits(_bits(fresh.eval(k8s.AUDIT_EP)), patched, "patch against a fresh upload")
    fresh.free()
    drv.close()
    return misses
