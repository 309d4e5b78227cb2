"""Lift the Cohere /v2/rerank vectors of the reference's tests into rerank_cases.json.

Usage: python extract_rerank_goldens.py <ai-gateway checkout>.  Sources:
  internal/translator/cohere_rerank_v2_test.go   TestCohereToCohereTranslatorV2Rerank_RequestBody (the four cases, with the
                                                 test's original body), _ResponseBody (the three cases; -1 = unset) and the
                                                 non_json_error / json_error_passthrough cases of _ResponseError
  internal/endpointspec/endpointspec_test.go     TestRerankEndpointSpec_ParseBody
The ParseBody success body is built by json.Marshal at run time; it is restated here as the bytes json.Marshal gives for
RerankV2Request{Model: "rerank-v3.5", Query: "foo", Documents: []string{"bar"}} (fields in struct order, the nil *int members
omitted)."""
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
GO_STR = r'(`[^`]*`|"(?:[^"\\]|\\.)*")'


def _go_string(lit):
    return lit[1:-1] if lit[0] == "`" else json.loads(lit)


def _func(src, name):
    at = src.index("func %s(" % name)
    end = src.find("\nfunc ", at + 1)
    return src[at:end if end > 0 else len(src)]


def _field(block, name, default=None):
    m = re.search(r"\b%s:\s*%s" % (name, GO_STR), block)
    if m:
        return _go_string(m.group(1))
    m = re.search(r"\b%s:\s*(-?\d+|true|false)" % name, block)
    return default if not m else {"true": True, "false": False}.get(m.group(1), None) if m.group(1) in ("true", "false") else int(m.group(1))


def _blocks(fn):
    """the case literals of a table-driven test: the text from one `name:` to the next"""
    at = [m.start() for m in re.finditer(r"\bname:\s", fn)]
    return [fn[a:b] for a, b in zip(at, at[1:] + [fn.index("} {", at[-1]) if "} {" in fn[at[-1]:] else len(fn)])]


def main(ref):
    tr = open(os.path.join(ref, "internal/translator/cohere_rerank_v2_test.go"), encoding="utf-8").read()
    fn = _func(tr, "TestCohereToCohereTranslatorV2Rerank_RequestBody")
    body = _go_string(re.search(r"originalBody := " + GO_STR, fn).group(1))
    version = _go_string(re.search(r'NewRerankCohereToCohereTranslator\(("[^"]*")', fn).group(1))
    request = [{"name": _field(b, "name"), "body": body, "version": version, "override": _field(b, "modelNameOverride", ""),
                "force": _field(b, "onRetry", False), "exp_path": _field(b, "expPath"), "exp_body_contains": _field(b, "expBodyContains", "")}
               for b in _blocks(fn)]
    fn = _func(tr, "TestCohereToCohereTranslatorV2Rerank_ResponseBody")
    response = [{"name": _field(b, "name"), "body": _field(b, "responseBody"), "error": _field(b, "expError", False),
                 "input": _field(b, "expectedInput", 0), "output": _field(b, "expectedOutput", 0), "total": _field(b, "expectedTotal", 0)}
                for b in _blocks(fn)]
    fn = _func(tr, "TestCohereToCohereTranslatorV2Rerank_ResponseError")
    errors = []
    for name in ("non_json_error", "json_error_passthrough"):
        b = fn[fn.index('t.Run("%s"' % name):]
        b = b[:b.index("\n\t})")]
        ct = re.search(r"contentTypeHeaderName:\s*(\"[^\"]*\"|jsonContentType)", b).group(1)
        errors.append({"name": name, "body": _go_string(re.search(r"errorBody := " + GO_STR, b).group(1)),
                       "content_type": "application/json" if ct == "jsonContentType" else _go_string(ct),
                       "status": _go_string(re.search(r"statusHeaderName:\s*(\"[^\"]*\")", b).group(1)),
                       "passthrough": "require.Nil(t, bodyMutation)" in b})
    es = open(os.path.join(ref, "internal/endpointspec/endpointspec_test.go"), encoding="utf-8").read()
    fn = _func(es, "TestRerankEndpointSpec_ParseBody")
    bad = _go_string(re.search(r"spec\.ParseBody\(\[\]byte\(" + GO_STR, fn).group(1))
    model = re.search(r'Model:\s*"([^"]*)", Query:\s*"([^"]*)", Documents:\s*\[\]string\{"([^"]*)"\}', fn)
    parse = [{"name": "invalid json", "body": bad, "error": True},
             {"name": "success", "body": json.dumps({"model": model.group(1), "query": model.group(2), "documents": [model.group(3)]}, separators=(",", ":")),
              "error": False, "model": model.group(1)}]
    out = {"source": "internal/translator/cohere_rerank_v2_test.go, internal/endpointspec/endpointspec_test.go (TestRerankEndpointSpec_ParseBody)",
           "request_body": request, "response_body": response, "response_error": errors, "parse_body": parse}
    with open(os.path.join(HERE, "rerank_cases.json"), "w", encoding="utf-8") as f:
        json.dump(out, f, indent=1, ensure_ascii=False)
    print(len(request), "request,", len(response), "response,", len(errors), "error,", len(parse), "parse cases")


if __name__ == "__main__":
    main(sys.argv[1])
