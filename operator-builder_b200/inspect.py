"""Host-side mirror of the BATCHED marker inspection (Go: operator-builder_b200/go/inspect_batch.go, workload_batch.go).

Reference today: one parser -- one lexer goroutine -- per YAML node, over Head + "\\n" + Line + "\\n" + Foot
(internal/markers/inspect/yaml.go:89-95, inspector.go:21-25), manifest by manifest
(internal/workload/v1/kinds/workload.go:224-228, :293-297).  Batched form, mirrored here:

    pass 1  walk every node of every manifest in the reference's visiting order and only collect the comment strings
    gpu     ONE Scanner.lex_batch over all of them
    pass 2  walk again in the same order; visit k parses the pre-lexed stream k (the parser is unchanged)

inspect_manifests_parsed does the same with ONE Scanner.parse_batch (scan and parser on the device): visit k formats the
Result records of input k.

What yaml.v3 attaches to which node as Head / Line / Foot comment is outside this path (it stays Go on the host, and no
reference test pins it): callers hand in the node tree with its comment strings.
"""
from typing import List, NamedTuple, Optional, Sequence

import numpy as np

from .lexer import Registry, Scanner, parse_doc_raw

MAPPING = "mapping"


class Node:
    """the part of yaml.v3's Node the walk looks at (yaml.go:62-107): Kind, Content, the three comments"""

    def __init__(self, kind: str = "scalar", content: Optional[Sequence["Node"]] = None, head: str = "", line: str = "", foot: str = ""):
        self.kind, self.content = kind, list(content) if content is not None else None
        self.head, self.line, self.foot = head, line, foot

    def comment_input(self) -> bytes:  # fmt.Sprintf("%s\n%s\n%s", ...), yaml.go:94
        return f"{self.head}\n{self.line}\n{self.foot}".encode("utf-8")


def visit(nodes: Sequence[Node], f):
    """inspectYAML (yaml.go:62-74): f(group, node) once per inspectYAMLComments node, in the reference's order"""
    for node in nodes:
        f((node,), node)
        if node.kind == MAPPING:
            visit_map(node.content or [], f)
        elif node.content is not None:
            visit(node.content, f)


def visit_map(nodes: Sequence[Node], f):
    """inspectYAMLMap (yaml.go:76-88): key/value pairs are one inspectYAMLComments call"""
    for i in range(0, len(nodes), 2):
        group = (nodes[i], nodes[i + 1])
        f(group, nodes[i])
        f(group, nodes[i + 1])
        if nodes[i + 1].kind == MAPPING:
            visit_map(nodes[i + 1].content or [], f)
        else:
            visit(nodes[i + 1].content or [], f)


class Collected(NamedTuple):
    docs: List[Node]
    inputs: List[bytes]


def collect(docs: Sequence[Node]) -> Collected:
    inputs: List[bytes] = []
    visit(docs, lambda _g, n: inputs.append(n.comment_input()))
    return Collected(list(docs), inputs)


def _pack(manifests: Sequence[Sequence[Node]]):
    """pass 1 over every manifest -> (collected, index of each manifest's first input, inputs, packed bytes, offsets)"""
    collected = [collect(m) for m in manifests]
    first, inputs = [], []
    for c in collected:
        first.append(len(inputs))
        inputs.extend(c.inputs)
    data = np.frombuffer(b"".join(inputs) + b"\0", dtype=np.uint8)[:-1] if inputs else np.zeros(0, np.uint8)
    off = np.zeros(len(inputs) + 1, dtype=np.uint64)
    if inputs:
        off[1:] = np.cumsum([len(x) for x in inputs])
    return collected, first, inputs, data, off


def _per_visit(collected, first, results_of):
    """pass 2: per manifest, (results_of(k), group) for visit k in visiting order"""
    out = []
    for c, k0 in zip(collected, first):
        k = [k0]
        per = []

        def one(group, node, k=k, per=per):
            per.append((results_of(k[0]), group))
            k[0] += 1

        visit(c.docs, one)
        out.append(per)
    return out


def inspect_manifests_batched(scanner: Scanner, registry: Registry, manifests: Sequence[Sequence[Node]]):
    """-> per manifest: list of (serialised parser Results of one visit, group) in visiting order.  One GPU call in all."""
    collected, first, inputs, data, off = _pack(manifests)
    res = scanner.lex_batch(data, off)
    return _per_visit(collected, first, lambda i: parse_doc_raw(registry, inputs[i], res.tuples[int(res.doc_tuple_off[i]):int(res.doc_tuple_off[i + 1])]))


def inspect_manifests_parsed(scanner: Scanner, registry: Registry, manifests: Sequence[Sequence[Node]]):
    """inspect_manifests_batched's result from ONE Scanner.parse_batch: the parser runs on the device too, and the host only
    formats the Result records (and parses the few nodes whose record says R_HOST from their returned tuples)."""
    collected, first, inputs, data, off = _pack(manifests)
    res = scanner.parse_batch(registry, data, off)
    return _per_visit(collected, first, lambda i: res.format_doc(i, inputs[i]))
