#!/usr/bin/env python3
"""Generate straight-line CUDA device code for AV1's 1-D butterfly networks.

Input : svt-av1-psy_b200/csrc/txfm_graphs.inc  (the networks as data, written by tools/extract_txfm_graphs.py)
Output: svt-av1-psy_b200/csrc/txfm_gen.inc     (one __device__ function per network: the whole vector in registers)

Each TXG_NODE(is_btf, wa, a, wb, b, clamp) becomes one SSA value; pure pass-through nodes (stage
permutations) cost nothing.  Two pruned 64-point variants are emitted as well: FDCT64_lo32 computes only
the 32 outputs the packed coefficient layout keeps (dead nodes dropped), IDCT64_in32 assumes inputs
32..63 are zero (zero operands folded: half_btf with one zero operand is a single product).  Arithmetic is the reference's: 32-bit wrapping add/sub, half_btf with
32-bit wrapping products summed in 64 bits (Source/Lib/Codec/inv_transforms.h:264).

Every function is a template on the cosine bit: `cosv` is a TxCosv<cos_bit> (txfm_tables.cuh), the cosine table of
that bit as a compile-time value, so each weight `cosv[k]` and each rounding shift of half_btf folds to an immediate
and no weight occupies a register.

Lane splits of the 32- and 64-point DCTs (the ones the fused kernel runs: FDCT32, FDCT64_lo32, IDCT32, IDCT64_in32):
the network's values after some stage fall into two groups whose cones share nothing but the inputs (which every
lane reads from shared memory).  split_plan() finds them by slicing the graph: it takes the largest stage count
`cut` at which the values fall into exactly two such groups.
  cut == all stages (forward DCT: even / odd outputs): <name>_g0 / _g1 compute the outputs of one group each;
  cut <  all stages (inverse DCT: the last stage combines the halves): <name>_g0 / _g1 compute the group's values
  after stage `cut`, and <name>_t0 / _t1 run the remaining stages from the whole cut vector to the outputs whose
  indices belong to that group.
struct TxgSplit_<name> gathers them with the element masks (bit i: element i) of what each one writes.
"""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "svt-av1-psy_b200", "csrc", "txfm_graphs.inc")
DST = os.path.join(ROOT, "svt-av1-psy_b200", "csrc", "txfm_gen.inc")


def parse(path):
    text = open(path).read()
    graphs = []
    for m in re.finditer(r"TXG_BEGIN\((\w+),\s*(\d+),\s*(\d+)\)(.*?)TXG_END\(\1\)", text, re.S):
        tag, n, st = m.group(1), int(m.group(2)), int(m.group(3))
        nodes = [tuple(int(v) for v in t.split(",")) for t in re.findall(r"TXG_NODE\(([^)]*)\)", m.group(4))]
        assert len(nodes) == n * st, (tag, len(nodes))
        graphs.append((tag, n, [nodes[s * n:(s + 1) * n] for s in range(st)]))
    return graphs


def emit(tag, n, stages, name=None, live_out=None, zero_in=None):
    """live_out: only these outputs are wanted (the rest of x[] is left untouched);
    zero_in: these inputs are known to be zero (constant-folded away)."""
    name = name or tag
    # backward liveness
    need = [None] * (len(stages) + 1)
    need[len(stages)] = set(range(n)) if live_out is None else set(live_out)
    for s in range(len(stages) - 1, -1, -1):
        cur_need = set()
        for i in need[s + 1]:
            btf, wa, a, wb, b, cl = stages[s][i]
            if wa:
                cur_need.add(a)
            if wb:
                cur_need.add(b)
        need[s] = cur_need
    out = []
    body = []
    cur = [None if (zero_in and i in zero_in) else "i%d" % i for i in range(n)]
    used_inputs = set()
    weights = set()
    for s, st in enumerate(stages):
        new = [None] * n
        for i, (btf, wa, a, wb, b, cl) in enumerate(st):
            if i not in need[s + 1]:
                new[i] = "/*dead*/0"
                continue
            nm = "s%d_%d" % (s, i)
            va, vb = (cur[a] if wa else None), (cur[b] if wb else None)
            for v in (va, vb):
                if v and v.startswith("i") and v[1:].isdigit():
                    used_inputs.add(int(v[1:]))
            if btf:
                W = lambda w: ("-c%d" % -w) if w < 0 else ("c%d" % w)
                if va is None and vb is None:
                    new[i] = None
                    continue
                if va is not None and vb is not None:
                    weights.update((abs(wa), abs(wb)))
                    expr = "txg_hbtf(%s, %s, %s, %s, cos_bit)" % (W(wa), va, W(wb), vb)
                elif va is not None:
                    weights.add(abs(wa))
                    expr = "txg_hbtf1(%s, %s, cos_bit)" % (W(wa), va)
                else:
                    weights.add(abs(wb))
                    expr = "txg_hbtf1(%s, %s, cos_bit)" % (W(wb), vb)
            else:
                assert wa in (-1, 0, 1) and wb in (-1, 0, 1)
                terms = [(w, v) for (w, v) in ((wa, va), (wb, vb)) if w and v is not None]
                if not terms:
                    new[i] = None  # zero (a clamp of zero is zero)
                    continue
                if len(terms) == 1 and terms[0][0] == 1 and not cl:
                    new[i] = terms[0][1]  # pass-through: no code
                    continue
                expr = "0u"
                for (w, v) in terms:
                    expr += " %s (uint32_t)%s" % ("+" if w > 0 else "-", v)
                expr = "(int32_t)(%s)" % expr
                if cl:
                    expr = "clamp_bits(%s, clampb)" % expr
            body.append("    const int32_t %s = %s;" % (nm, expr))
            new[i] = nm
        cur = new
    out.append("template <int cos_bit>")
    out.append("__device__ __forceinline__ void txg_%s(int32_t (&x)[%d], TxCosv<cos_bit> cosv, const int clampb) {" % (name, n))
    out.append("    (void)clampb;")
    for w in sorted(weights):
        out.append("    const int32_t c%d = cosv[%d];" % (w, w))
    for i in sorted(used_inputs):
        out.append("    const int32_t i%d = x[%d];" % (i, i))
    out += body
    for i in sorted(need[len(stages)]):
        out.append("    x[%d] = %s;" % (i, cur[i] if cur[i] is not None else "0"))
    out.append("}")
    return "\n".join(out)


def split_plan(n, stages):
    """(cut, [group0, group1]): see the module docstring.  Groups are sorted element-index lists."""
    for cut in range(len(stages), 0, -1):
        parent = {}

        def find(v):
            while parent.setdefault(v, v) != v:
                v = parent[v]
            return v

        cur = [("in", i) for i in range(n)]
        for s in range(cut):
            new = []
            for i, (btf, wa, a, wb, b, cl) in enumerate(stages[s]):
                me = (s, i)
                find(me)
                for w, o in ((wa, a), (wb, b)):
                    if w and cur[o][0] != "in":  # inputs are shared read-only leaves: they do not join groups
                        parent[find(me)] = find(cur[o])
                new.append(me)
            cur = new
        groups = {}
        for i, v in enumerate(cur):
            groups.setdefault(find(v), []).append(i)
        if len(groups) >= 2:
            assert len(groups) == 2, "split into %d groups" % len(groups)
            return cut, sorted((sorted(g) for g in groups.values()), key=lambda g: g[0])
    raise ValueError("network does not split")


# the networks the fused kernel runs split across two lanes: (emitted name, graph tag, live outputs, zero inputs)
SPLITS = (("FDCT32", "FDCT32", None, None),
          ("FDCT64_lo32", "FDCT64", range(32), None),
          ("IDCT32", "IDCT32", None, None),
          ("IDCT64_in32", "IDCT64", None, set(range(32, 64))))


def split_functions(n, stages, name, live_out=None, zero_in=None):
    """[(function name, stage range, live outputs of the function)] of the split of one network"""
    cut, groups = split_plan(n, stages)
    live = set(range(n)) if live_out is None else set(live_out)
    fns = []
    for k, g in enumerate(groups):
        if cut == len(stages):
            fns.append(("%s_g%d" % (name, k), (0, cut), sorted(set(g) & live)))
        else:
            fns.append(("%s_g%d" % (name, k), (0, cut), list(g)))
            fns.append(("%s_t%d" % (name, k), (cut, len(stages)), sorted(set(g) & live)))
    return cut, fns


def emit_split(n, stages, name, live_out=None, zero_in=None):
    """the split's functions, then struct TxgSplit_<name>: kTail, the masks kMid<k> (what _g<k> writes) and kOut<k>
    (the outputs lane group k stores), mid<k>() / tail<k>() dispatching to the functions"""
    cut, fns = split_functions(n, stages, name, live_out, zero_in)
    out = []
    for fn, (s0, s1), live in fns:
        out.append(emit(fn, n, stages[s0:s1], name=fn, live_out=live, zero_in=zero_in if s0 == 0 else None))
        out.append("")
    mask = {fn: "0x%016xull" % sum(1 << i for i in live) for fn, _, live in fns}
    tail = cut < len(stages)
    sig = "(int32_t (&x)[%d], TxCosv<cos_bit> cosv, const int clampb)" % n
    out.append("struct TxgSplit_%s {" % name)
    out.append("    static constexpr bool kTail = %s;" % ("true" if tail else "false"))
    for k in range(2):
        out.append("    static constexpr unsigned long long kMid%d = %s, kOut%d = %s;" %
                   (k, mask["%s_g%d" % (name, k)], k, mask["%s_%s%d" % (name, "t" if tail else "g", k)]))
    for part, letter in (("mid", "g"), ("tail", "t")) if tail else (("mid", "g"),):
        out.append("    template <int G, int cos_bit> static __device__ __forceinline__ void %s%s {" % (part, sig))
        out.append("        if constexpr (G == 0) txg_%s_%s0(x, cosv, clampb); else txg_%s_%s1(x, cosv, clampb);" %
                   (name, letter, name, letter))
        out.append("    }")
    out.append("};")
    out.append("")
    return "\n".join(out)


def main():
    graphs = parse(SRC)
    parts = ["// GENERATED by tools/gen_txfm_code.py from txfm_graphs.inc -- do not edit.",
             "// Straight-line register versions of the 1-D networks (one thread = one vector).", ""]
    for tag, n, stages in graphs:
        parts.append(emit(tag, n, stages))
        parts.append("")
        if tag == "FDCT64":  # packed output: only the 32 low-frequency coefficients are kept (transforms.c:2374)
            parts.append(emit(tag, n, stages, name="FDCT64_lo32", live_out=range(32)))
            parts.append("")
        if tag == "IDCT64":  # packed input: coefficients 32..63 are zero (inv_transforms.c:2567-2686)
            parts.append(emit(tag, n, stages, name="IDCT64_in32", zero_in=set(range(32, 64))))
            parts.append("")
    by_tag = {tag: (n, stages) for tag, n, stages in graphs}
    parts.append("// Two-lane splits (see tools/gen_txfm_code.py)")
    for name, tag, live_out, zero_in in SPLITS:
        n, stages = by_tag[tag]
        parts.append(emit_split(n, stages, name, live_out, zero_in))
    open(DST, "w").write("\n".join(parts))
    print("wrote", DST, "(%d networks)" % len(graphs))


if __name__ == "__main__":
    main()
