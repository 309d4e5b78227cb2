"""Lift the /v1/responses response-side vectors of the reference's translator tests into responses_cases.json.

Usage: python extract_responses_goldens.py <ai-gateway checkout>.  Source: internal/translator/openai_responses_test.go
(TestResponses_HandleStreamingResponse, TestResponses_HandleNonStreamingResponse, TestResponses_ExtractUsageFromBufferEvent).
Usage rows are (input, output, total, cached, cache_creation, reasoning) with -1 for a counter the call leaves unset."""
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def main(ref):
    src = open(os.path.join(ref, "internal/translator/openai_responses_test.go"), encoding="utf-8").read()

    def block(run_name, var):
        at = src.index('t.Run("%s"' % run_name)
        m = re.compile(var + r" := (?:\[\]byte\()?`(.*?)`", re.S).search(src, at)
        return m.group(1)

    full = block("valid streaming events", "sseChunks")
    streams = [
        {"name": "valid streaming events", "data": full, "request_model": "gpt-4o",
         "exp": [10, 5, 15, 2, 0, 0], "exp_model": "gpt-4o-2024-11-20"},
        {"name": "valid usage data", "data": block("valid usage data", "chunks"), "request_model": "",
         "exp": [10, 5, 15, 2, 0, 0], "exp_model": "gpt-4o-2024-11-20"},
        {"name": "model extraction", "data": block("model extraction", "chunks"), "request_model": "",
         "exp": None, "exp_model": "gpt-4o-2024-11-20"},
        {"name": "invalid JSON skipped", "data": block("invalid JSON skipped", "chunks"), "request_model": "",
         "exp": [5, 3, 8, 0, 0, 0], "exp_model": ""},
        {"name": "no usage data", "data": block("no usage data", "chunks"), "request_model": "",
         "exp": [-1, -1, -1, -1, -1, -1], "exp_model": "gpt-4o"},
    ]
    buffered = [
        {"name": "complete response", "body": block("complete response", "respJSON"), "exp_error": False,
         "exp": [10, 5, 15, 2, 0, 0], "exp_model": "gpt-4o-2024-11-20"},
        {"name": "invalid JSON", "body": "{invalid json", "exp_error": True},
    ]
    with open(os.path.join(HERE, "responses_cases.json"), "w", encoding="utf-8") as f:
        json.dump({"source": "internal/translator/openai_responses_test.go:517-811", "streams": streams, "buffered": buffered}, f, indent=1)


if __name__ == "__main__":
    main(sys.argv[1])
