"""Lift the /v1/responses request-side vectors of the reference's tests into responses_request_cases.json.

Usage: python extract_responses_request_goldens.py <ai-gateway checkout>.  Sources:
  internal/apischema/openai/openai_test.go   the UnmarshalJSON tables of the request unions: each case's JSON and whether it errors
  internal/endpointspec/endpointspec_test.go TestResponsesEndpointSpec_ParseBody
  internal/translator/openai_responses_test.go TestResponsesOpenAIToOpenAITranslator_RequestBody (override, stream, forced mutation)
Each union case is also wrapped into the request member that decodes it ("wrapped"), so that the request decode can be checked."""
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
UNIONS = {   # test → how a value of that union sits in a request body
    "TestResponseNewParamsInputUnionUnmarshalJSON": '{"model":"m","input":%s}',
    "TestResponseInputItemUnionParamUnmarshalJSON": '{"model":"m","input":[%s]}',
    "TestResponseInputContentUnionParamUnmarshalJSON": '{"model":"m","input":[{"role":"user","content":[%s]}]}',
    "TestResponseToolUnionUnmarshalJSON": '{"model":"m","tools":[%s]}',
    "TestResponseToolChoiceUnionUnmarshalJSON": '{"model":"m","tool_choice":%s}',
    "TestResponseFormatTextConfigUnionParamUnmarshalJSON": '{"model":"m","text":{"format":%s}}',
    "TestResponseNewParamsConversationUnionUnmarshalJSON": '{"model":"m","conversation":%s}',
}
CASE = re.compile(r'\n\t\t\{\n(.*?)\n\t\t\},', re.S)
JSON = re.compile(r'(?:input|data|json|jsonStr|jsonData)\s*:\s*(?:\[\]byte\()?(`[^`]*`|"(?:[^"\\]|\\.)*")')
ERR = re.compile(r'(?:expErr|wantErr|expectErr|expectedErr|expError|errContains)\s*:\s*(true|"[^"]+")')


def _go_string(lit):
    return lit[1:-1] if lit[0] == "`" else json.loads(lit)


def _func(src, name):
    at = src.find("func %s(" % name)
    if at < 0:
        return None
    end = src.find("\nfunc ", at + 1)
    return src[at:end if end > 0 else len(src)]


def main(ref):
    src = open(os.path.join(ref, "internal/apischema/openai/openai_test.go"), encoding="utf-8").read()
    unions = []
    for test, wrap in UNIONS.items():
        body = _func(src, test)
        if body is None:
            continue
        for m in CASE.finditer(body):
            c = m.group(1)
            name = re.search(r'name:\s*"([^"]*)"', c)
            js = JSON.search(c)
            if not name or not js:
                continue
            val = _go_string(js.group(1))
            unions.append({"test": test, "name": name.group(1), "json": val, "error": bool(ERR.search(c)), "wrapped": wrap % val})
    parse = [
        {"name": "invalid json", "body": "{", "error": True},
        {"name": "success", "body": '{"model":"gpt-4o","input":"Hi","stream":true}', "error": False, "model": "gpt-4o", "stream": True},
        {"name": "array_input_without_type_field", "error": False, "model": "gpt-4.7", "stream": False,
         "body": '{\n\t\t\t"model": "gpt-4.7",\n\t\t\t"input": [{"role": "user", "content": "Hello"}],\n\t\t\t"max_tokens": 50\n\t\t}'},
    ]
    request = [   # exp_body: null = no body; "original" = the input bytes; exp_model_member = the model the body must carry
        {"name": "basic request without override", "body": '{"model":"gpt-4o","input":"Hi"}', "override": "", "force": False, "exp_path": "/v1/responses", "exp_body": None},
        {"name": "streaming request", "body": '{"model":"gpt-4o","stream":true,"input":"Hi"}', "override": "", "force": False, "exp_path": "/v1/responses", "exp_body": None, "stream": True},
        {"name": "model name override", "body": '{"model":"gpt-4o","input":"Hi"}', "override": "gpt-4-turbo", "force": False, "exp_path": "/v1/responses", "exp_model_member": "gpt-4-turbo"},
        {"name": "forced mutation without override", "body": '{"model":"gpt-4o", "input":"Hi"}', "override": "", "force": True, "exp_path": "/v1/responses", "exp_body": "original"},
    ]
    out = {"source": "internal/apischema/openai/openai_test.go (request-union UnmarshalJSON tables), internal/endpointspec/endpointspec_test.go:294-334, "
                     "internal/translator/openai_responses_test.go:48-164",
           "unions": unions, "parse_body": parse, "request_body": request}
    with open(os.path.join(HERE, "responses_request_cases.json"), "w", encoding="utf-8") as f:
        json.dump(out, f, indent=1)
    print(len(unions), "union cases")


if __name__ == "__main__":
    main(sys.argv[1])
