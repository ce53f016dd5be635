"""Gate graphs as the reference stores them (gates.xsd; written by save_state, state.c:107-166):
a loader that needs no libxml2, and an independent functional check.

`load_graph` does what load_state does (state.c:260-411): reads the gates in order, enforces the
same structural rules, and recomputes every gate's 256-bit truth table from the topology.
`verify_graph` then compares each output gate's table with the S-box bit it claims to compute
(sboxgates.c:745) -- a check that does not depend on anything the search code did.  Used by the
test-suite and bench.py on the files the GPU build writes.
"""
import xml.etree.ElementTree as ET
from dataclasses import dataclass, field
from typing import List

import numpy as np

MASK256 = (1 << 256) - 1

# state.h:35-56 / state.c:33-53; a two-input gate type's number is its truth table over (A, B):
# bit ((1 - A) << 1 | (1 - B)) of the number is the output (AND = 1, NOR = 8; boolfunc.c:136-157).
GATE_NAMES = ["FALSE", "AND", "A_AND_NOT_B", "A", "NOT_A_AND_B", "B", "XOR", "OR", "NOR", "XNOR",
              "NOT_B", "A_OR_NOT_B", "NOT_A", "NOT_A_OR_B", "NAND", "TRUE", "NOT", "IN", "LUT"]
NO_GATE = 0xFFFF


@dataclass
class Gate:
    type: str
    inputs: List[int]
    function: int = 0
    table: int = 0       # 256-bit truth table as an int: bit p = value at S-box input p


@dataclass
class Graph:
    gates: List[Gate] = field(default_factory=list)
    outputs: dict = field(default_factory=dict)   # output bit -> gate number

    @property
    def num_inputs(self):
        return sum(1 for g in self.gates if g.type == "IN")

    @property
    def num_luts(self):
        return sum(1 for g in self.gates if g.type == "LUT")


class GraphError(ValueError):
    pass


def input_table(bit):
    """generate_target(bit, false) (state.c:232-250): position p holds bit `bit` of p."""
    t = 0
    for p in range(256):
        if (p >> bit) & 1:
            t |= 1 << p
    return t


def sbox_table(sbox, bit):
    """generate_target(bit, true): position p holds bit `bit` of sbox[p]."""
    t = 0
    for p in range(256):
        if (sbox[p] >> bit) & 1:
            t |= 1 << p
    return t


def lut_table(func, a, b, c):
    """generate_lut_ttable (state.c:202-230): function bit index = in1 << 2 | in2 << 1 | in3."""
    out = 0
    for m in range(8):
        if (func >> m) & 1:
            out |= (a if m & 4 else ~a) & (b if m & 2 else ~b) & (c if m & 1 else ~c)
    return out & MASK256


def gate2_table(type_index, a, b):
    """generate_ttable_2 (boolfunc.c:136-157)."""
    out = 0
    for m in range(4):
        if (type_index >> m) & 1:
            out |= (~a if m & 2 else a) & (~b if m & 1 else b)
    return out & MASK256


def load_graph(path):
    """Parses a gates.xsd file with the checks of load_state (state.c:260-411)."""
    try:
        root = ET.parse(path).getroot()
    except ET.ParseError as exc:
        raise GraphError("not well-formed XML: %s" % exc) from exc
    if root.tag != "gates":
        raise GraphError("root element is <%s>, expected <gates>" % root.tag)
    g = Graph()
    for el in root:
        if el.tag != "gate":
            continue
        typ = el.get("type")
        if typ not in GATE_NAMES:
            raise GraphError("unknown gate type %r" % typ)
        func = 0
        if el.get("function") is not None:
            func = int(el.get("function"), 16)
            if func <= 0 or func > 255:
                raise GraphError("LUT function out of range")
        if typ != "LUT" and func != 0:
            raise GraphError("function attribute on a %s gate" % typ)
        inputs = []
        for inp in el:
            if inp.tag != "input":
                continue
            num = int(inp.get("gate"))
            if num >= len(g.gates):
                raise GraphError("gate %d uses gate %d, which does not precede it" % (len(g.gates), num))
            inputs.append(num)
        idx = GATE_NAMES.index(typ)
        if idx <= 15:
            if len(inputs) != 2:
                raise GraphError("two-input gate with %d inputs" % len(inputs))
            table = gate2_table(idx, g.gates[inputs[0]].table, g.gates[inputs[1]].table)
        elif typ == "NOT":
            if len(inputs) != 1:
                raise GraphError("NOT gate with %d inputs" % len(inputs))
            table = ~g.gates[inputs[0]].table & MASK256
        elif typ == "IN":
            if inputs or len(g.gates) >= 8 or (g.gates and g.gates[-1].type != "IN"):
                raise GraphError("misplaced IN gate")
            table = input_table(len(g.gates))
        else:
            if len(inputs) != 3:
                raise GraphError("LUT with %d inputs" % len(inputs))
            table = lut_table(func, *(g.gates[i].table for i in inputs))
        g.gates.append(Gate(typ, inputs, func, table))
        if len(g.gates) > 500:
            raise GraphError("more than MAX_GATES gates")
    for el in root:
        if el.tag != "output":
            continue
        bit, gate = int(el.get("bit")), int(el.get("gate"))
        if bit >= 8 or bit in g.outputs or gate >= len(g.gates):
            raise GraphError("bad output element")
        g.outputs[bit] = gate
    return g


def gate_depths(graph):
    """The depth of every gate of a loaded graph, in gate order, as a numpy uint16 array: 0 for an
    input, else 1 + the largest depth among the gate's inputs.  What LutEngine.set_depth_filter
    takes for the graph's search state."""
    depth = np.zeros(len(graph.gates), dtype=np.uint16)
    for i, g in enumerate(graph.gates):
        if g.type != "IN":
            depth[i] = 1 + max((int(depth[j]) for j in g.inputs), default=0)
    return depth


def verify_graph(graph, sbox, require_bits=None):
    """Every output gate computes its S-box bit on all 2^num_inputs inputs (sboxgates.c:745).
    Returns the list of verified output bits; raises GraphError otherwise."""
    if not graph.outputs:
        raise GraphError("graph has no outputs")
    n_in = graph.num_inputs
    care = 0
    for p in range(1 << n_in):
        care |= 1 << p
    for bit, gate in sorted(graph.outputs.items()):
        if (graph.gates[gate].table ^ sbox_table(sbox, bit)) & care:
            raise GraphError("output bit %d: gate %d does not compute the S-box bit" % (bit, gate))
    if require_bits is not None and sorted(graph.outputs) != sorted(require_bits):
        raise GraphError("outputs %s, expected %s" % (sorted(graph.outputs), sorted(require_bits)))
    return sorted(graph.outputs)


def load_sbox(path):
    """load_sbox (sboxgates.c:992-1040): whitespace-separated hex bytes; returns the 256-entry table
    (shorter tables padded with zeros) and the number of entries read."""
    vals = [int(tok, 16) for tok in open(path).read().split()]
    if not vals or len(vals) > 256 or any(v > 255 for v in vals):
        raise GraphError("bad S-box file")
    return vals + [0] * (256 - len(vals)), len(vals)
