#!/usr/bin/env python
"""Writes tests/golden/predicted_results_handmade.json: every {"itemScores":[...]} line that the deployed reference engine
served in its integration tests, transcribed from data/integration-test-expected.txt, data/integration-test-item-set-
expected.txt and data/rank-test-query-expected.txt of the reference project, each with its file and 1-based line number.
The scores keep ES's own text (0.18232156, 0.3595937192440033).  Usage: make_predicted_results_fixture.py <reference
checkout>.  The tests synthesise one _msearch response element per line from it: hits in that order, _score written with
exactly the line's score text, _source from item_queries_handmade.json's index where the item has a document.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
FILES = ["data/integration-test-expected.txt", "data/integration-test-item-set-expected.txt", "data/rank-test-query-expected.txt"]


def main(ref: str) -> None:
    lines = []
    for f in FILES:
        for n, line in enumerate(open(os.path.join(ref, f), encoding="utf-8"), 1):
            if line.startswith('{"itemScores"'):
                lines.append({"file": f, "line": n, "text": line.rstrip("\n")})
    out = {"source": "the PredictedResult lines of the reference's integration tests (see the generator)", "results": lines}
    with open(os.path.join(HERE, "predicted_results_handmade.json"), "w", encoding="utf-8") as fh:
        json.dump(out, fh, indent=1, ensure_ascii=False)
        fh.write("\n")
    print(f"{len(lines)} lines")


if __name__ == "__main__":
    main(sys.argv[1])
