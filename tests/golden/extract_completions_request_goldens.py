"""Lift the /v1/completions request-side vectors of the reference's tests into completions_request_cases.json.

Usage: python extract_completions_request_goldens.py <ai-gateway checkout>.  Sources:
  internal/apischema/openai/union_test.go        TestUnmarshalJSONNestedUnion (its extra success cases) and _Errors
  internal/apischema/openai/openai_bench_test.go promptUnionBenchmarkCases (success cases of TestUnmarshalJSONNestedUnion too)
  internal/endpointspec/endpointspec_test.go     TestCompletionsEndpointSpec_ParseBody
  internal/translator/openai_completions_test.go TestOpenAIToOpenAITranslatorV1CompletionRequestBody / …Streaming
  tests/internal/testopenai/cassettes/completion-*.yaml   the recorded request bodies (checked against content_length)
Each prompt-union case is wrapped as {"model":"m","prompt":<data>}; cases whose wrapped body is not JSON (the truncated ones) are
skipped, since the request decoder rejects them before the union sees them."""
import glob
import json
import os
import re
import sys

import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
WRAP = '{"model":"m","prompt":%s}'
CASE = re.compile(r'name:\s*"([^"]*)",[^\n]*\n\s*data:\s*\[\]byte(?:\((`[^`]*`|"(?:[^"\\]|\\.)*")\)|\{\})')


def _go_string(lit):
    return lit[1:-1] if lit[0] == "`" else json.loads(lit)


def _func(src, name):
    at = src.find("func %s(" % name)
    end = src.find("\nfunc ", at + 1)
    return src[at:end if end > 0 else len(src)]


def _cases(text, test, error):
    out = []
    for m in CASE.finditer(text):
        data = _go_string(m.group(2)) if m.group(2) else ""
        wrapped = WRAP % data
        try:
            json.loads(wrapped)
        except ValueError:
            continue
        out.append({"test": test, "name": m.group(1), "json": data, "error": error, "wrapped": wrapped})
    return out


def main(ref):
    union = open(os.path.join(ref, "internal/apischema/openai/union_test.go"), encoding="utf-8").read()
    bench = open(os.path.join(ref, "internal/apischema/openai/openai_bench_test.go"), encoding="utf-8").read()
    at = bench.index("promptUnionBenchmarkCases = []struct")
    unions = _cases(bench[at:bench.index("contentUnionBenchmarkCases", at)], "promptUnionBenchmarkCases", False)
    unions += _cases(_func(union, "TestUnmarshalJSONNestedUnion"), "TestUnmarshalJSONNestedUnion", False)
    unions += _cases(_func(union, "TestUnmarshalJSONNestedUnion_Errors"), "TestUnmarshalJSONNestedUnion_Errors", True)
    parse = [   # the streaming case marshals openai.CompletionRequest{Model, Stream: true, Prompt: "say hi"}: fields in struct order
        {"name": "invalid json", "body": "{bad", "error": True},
        {"name": "streaming", "body": '{"model":"text-davinci-003","prompt":"say hi","stream":true}', "error": False, "model": "text-davinci-003", "stream": True},
    ]
    body = '{"model":"gpt-3.5-turbo-instruct","prompt":"Say hello","max_tokens":10}'
    request = [   # exp_body: null = no body; "original" = the input bytes; exp_model_member = the model the body must carry
        {"name": "valid_body", "body": body, "override": "", "force": False, "exp_path": "/v1/completions", "exp_body": None},
        {"name": "model_name_override", "body": body, "override": "custom-completion-model", "force": False, "exp_path": "/v1/completions",
         "exp_model_member": "custom-completion-model"},
        {"name": "on_retry", "body": body, "override": "", "force": True, "exp_path": "/v1/completions", "exp_body": "original"},
        {"name": "model_name_override_with_retry", "body": body, "override": "custom-completion-model", "force": True, "exp_path": "/v1/completions",
         "exp_model_member": "custom-completion-model"},
        {"name": "streaming", "body": '{"model":"gpt-3.5-turbo-instruct","prompt":"Say hello","stream":true}', "override": "", "force": False,
         "exp_path": "/v1/completions", "exp_body": None, "stream": True},
    ]
    cassettes = []
    for path in sorted(glob.glob(os.path.join(ref, "tests/internal/testopenai/cassettes/completion-*.yaml"))):
        req = yaml.safe_load(open(path, encoding="utf-8"))["interactions"][0]["request"]
        assert len(req["body"].encode()) == req["content_length"], path
        cassettes.append({"name": os.path.basename(path)[:-5], "body": req["body"], "content_length": req["content_length"]})
    out = {"source": "internal/apischema/openai/union_test.go:18-167, openai_bench_test.go (promptUnionBenchmarkCases), "
                     "internal/endpointspec/endpointspec_test.go:106-126, internal/translator/openai_completions_test.go:20-98, "
                     "tests/internal/testopenai/cassettes/completion-*.yaml",
           "unions": unions, "parse_body": parse, "request_body": request, "cassettes": cassettes}
    with open(os.path.join(HERE, "completions_request_cases.json"), "w", encoding="utf-8") as f:
        json.dump(out, f, indent=1, ensure_ascii=False)
    print(len(unions), "union cases,", len(cassettes), "cassettes")


if __name__ == "__main__":
    main(sys.argv[1])
