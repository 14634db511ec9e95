"""Row / column structure of a grid region: `parse_grid_from_bottom_up` (reference src/yomitoku/grid_parser.py:1-923).

The cells of a region become nodes of an adjacency graph with R / L / D / U edges; every cell that borders several
cells on one side is split into unit cells, one per neighbour ("dup" nodes); the rows are the R-chains from the heads
of the rows and the columns the D-chains, and each grid position holds the cell that lies on both.  Header rows (only
header / empty cells) give the column headers.  Host code like in the reference; the graph is a networkx DiGraph
whose node and edge orders are the reference's, since they decide the splits.
"""
from collections import deque
from itertools import count

import networkx as nx

from .document_analyzer import is_bottom_adjacent, is_right_adjacent
from .schemas import TableGridSchema

__all__ = ["parse_grid_from_bottom_up", "adjacency_thresholds", "line_from_head"]

# adjacency thresholds relative to the cell size (reference :16-27): a fixed pixel distance either skips a thin row or
# misses a thick one; the scale is the lower quartile of the cell heights and widths
DIST_SCALE, IGNORE_SCALE, DIST_FLOOR = 0.5, 0.25, 3.0
# two neighbours on the split side whose intervals overlap this much (IoU) are one detection seen twice (:111-115)
SAME_SLOT_IOU = 0.7


def _lower_quartile(values):
    vals = sorted(values)
    return vals[min(int(len(vals) * 0.25), len(vals) - 1)]


def adjacency_thresholds(boxes):
    """{"dist", "ignore"}: the adjacency distance and the diagonal-contact distance for cells of these sizes
    (reference :30-63)."""
    if not boxes:
        return {"dist": DIST_FLOOR, "ignore": DIST_FLOOR / 2}
    scale = min(_lower_quartile([b[3] - b[1] for b in boxes]), _lower_quartile([b[2] - b[0] for b in boxes]))
    return {"dist": max(DIST_FLOOR, DIST_SCALE * scale), "ignore": max(DIST_FLOOR / 2, IGNORE_SCALE * scale)}


def _adj_kwargs(th):
    return dict(dist_threshold=th["dist"], ignore_dist_threshold=th["ignore"], overlap_ratio_th=0.25)


def _grid_graph(nodes, th):
    """Cells, empties and headers as nodes; both directions of every soft adjacency as edges (reference :66-108)."""
    g = nx.DiGraph()
    cells = nodes["cell"] + nodes["empty"] + nodes["header"]
    for c in cells:
        g.add_node(c.id, bbox=c.box, role=c.role, contents=c.contents)
    kw = _adj_kwargs(th)
    for a in cells:
        for b in cells:
            if a.id == b.id:
                continue
            if is_bottom_adjacent(a.box, b.box, **kw):
                g.add_edge(a.id, b.id, dir="D")
                g.add_edge(b.id, a.id, dir="U")
            if is_right_adjacent(a.box, b.box, **kw):
                g.add_edge(a.id, b.id, dir="R")
                g.add_edge(b.id, a.id, dir="L")
    return g


def _slot_groups(g, outs, axis):
    """Neighbours grouped by near-identical intervals on `axis` (union-find over pairs with IoU >= SAME_SLOT_IOU),
    groups and their interval hulls in the order of the hull centres (reference :118-167)."""
    ivs = [(g.nodes[n]["bbox"][axis], g.nodes[n]["bbox"][axis + 2]) for n in outs]
    parent = list(range(len(outs)))

    def root(i):
        while parent[i] != i:
            parent[i] = parent[parent[i]]
            i = parent[i]
        return i

    for i in range(len(outs)):
        for j in range(i + 1, len(outs)):
            inter = max(0.0, min(ivs[i][1], ivs[j][1]) - max(ivs[i][0], ivs[j][0]))
            union = max(ivs[i][1], ivs[j][1]) - min(ivs[i][0], ivs[j][0])
            if union > 0 and inter / union >= SAME_SLOT_IOU:
                parent[root(i)] = root(j)
    members = {}
    for i in range(len(outs)):
        members.setdefault(root(i), []).append(i)
    groups = [[outs[i] for i in m] for m in members.values()]
    hulls = [(min(ivs[i][0] for i in m), max(ivs[i][1] for i in m)) for m in members.values()]
    order = sorted(range(len(groups)), key=lambda k: (hulls[k][0] + hulls[k][1]) / 2.0)
    return [groups[k] for k in order], [hulls[k] for k in order]


def _slots(lo, hi, groups, hulls, min_len):
    """[lo, hi] cut into consecutive slots along the ordered group hulls; a group left with no more than min_len of
    its own joins the slot before it (or the next one when it comes first); the last slot reaches hi
    (reference :170-217).  Returns (segments, groups per segment)."""
    segs, merged, pending, cur = [], [], [], lo
    for group, (a, b) in zip(groups, hulls):
        a = max(max(lo, min(a, hi)), cur)
        b = max(max(lo, min(b, hi)), a)
        if b - a <= min_len:
            (merged[-1] if merged else pending).extend(group)
            continue
        merged.append(pending + list(group))
        pending = []
        segs.append([a, b])
        cur = b
    if pending and merged:
        merged[-1].extend(pending)
    if segs:
        segs[-1][1] = hi
    return segs, merged


# The two split passes of reference :220-502: `fwd` is the side whose several neighbours split the node, `chain` the
# perpendicular direction the pieces are chained along.  Rows: fwd R (then L), pieces stacked with D; columns: fwd D
# (then U), pieces side by side with R.
_SPLIT = {
    "R": dict(back="L", axis=1, chain="D", rev_chain="U"),
    "L": dict(back="R", axis=1, chain="D", rev_chain="U"),
    "D": dict(back="U", axis=0, chain="R", rev_chain="L"),
    "U": dict(back="D", axis=0, chain="R", rev_chain="L"),
}


def _split_from_head(dag, head, fwd, th):
    """Walks the graph breadth-first from `head` along `fwd` edges and splits every node with more than one slot of
    `fwd` neighbours into one piece per slot (reference normalize_row_with_out_edges :220-367 and
    normalize_col_with_out_edges :370-502)."""
    spec = _SPLIT[fwd]
    back, axis, chain, rev_chain = spec["back"], spec["axis"], spec["chain"], spec["rev_chain"]
    kw = _adj_kwargs(th)
    g = dag.copy()
    queue = deque([head])
    serial = count(1)

    def back_adjacent(bwd, piece):
        pb, bb = g.nodes[piece]["bbox"], g.nodes[bwd]["bbox"]
        if fwd == "R":
            return is_right_adjacent(bb, pb, **kw)
        if fwd == "L":
            return is_right_adjacent(pb, bb, **kw)
        if fwd == "D":
            return is_bottom_adjacent(bb, pb, **kw)
        return is_bottom_adjacent(pb, bb, **kw)

    while queue:
        u = queue.popleft()
        if u not in g.nodes:
            continue
        outs = [v for v in g.successors(u) if g[u][v].get("dir") == fwd]
        # the cells behind u: for R / L / D the predecessors that point at u with `fwd`; for U (the reference's column
        # pass run backwards) the successors u points at with D
        if fwd == "U":
            behind = [v for v in g.successors(u) if g[u][v].get("dir") == "D"]
        else:
            behind = [p for p in g.predecessors(u) if g[p][u].get("dir") == fwd]
        before = [p for p in g.predecessors(u) if g[p][u].get("dir") == chain]     # above u (rows) / left of u (cols)
        after = [v for v in g.successors(u) if g[u][v].get("dir") == chain]        # below u / right of u
        slot_groups = []
        if len(outs) > 1:
            groups, hulls = _slot_groups(g, outs, axis)
            box = g.nodes[u]["bbox"]
            segs, slot_groups = _slots(box[axis], box[axis + 2], groups, hulls, th["ignore"])
        if len(slot_groups) <= 1:
            queue.extend(outs)
            continue
        x1, y1, x2, y2 = g.nodes[u]["bbox"]
        attrs = dict(g.nodes[u])
        pieces = []
        for a, b in segs:
            name = "%s__dup%d" % (u, next(serial))
            g.add_node(name, **dict(attrs, bbox=(x1, a, x2, b) if axis == 1 else (a, y1, b, y2)))
            pieces.append(name)
        for group, piece in zip(slot_groups, pieces):
            for v in group:
                g.add_edge(piece, v, dir=fwd)
                g.add_edge(v, piece, dir=back)
        for p in before:
            g.add_edge(pieces[0], p, dir=rev_chain)
            g.add_edge(p, pieces[0], dir=chain)
        for p in after:
            g.add_edge(pieces[-1], p, dir=chain)
            g.add_edge(p, pieces[-1], dir=rev_chain)
        for a, b in zip(pieces, pieces[1:]):
            g.add_edge(a, b, dir=chain)
            g.add_edge(b, a, dir=rev_chain)
        for bwd in behind:
            for piece in pieces:
                if back_adjacent(bwd, piece):
                    g.add_edge(bwd, piece, dir=fwd)
                    g.add_edge(piece, bwd, dir=back)
                    queue.append(bwd)
        g.remove_node(u)
        queue.extend(pieces)
    return g


def _heads(dag, direction):
    """The start nodes of the `direction` chains: per connected component of the `direction` edges (isolated nodes
    included, components in node order) its nodes without an incoming `direction` edge, sorted, or else its smallest
    node (reference :541-574)."""
    und = nx.Graph()
    und.add_nodes_from(dag.nodes())
    und.add_edges_from((u, v) for u, v, d in dag.edges(data=True) if d.get("dir") == direction)
    sub = nx.DiGraph((u, v, d) for u, v, d in dag.edges(data=True) if d.get("dir") == direction)
    sub.add_nodes_from(dag.nodes())
    heads = []
    for comp in nx.connected_components(und):
        roots = [n for n in comp if sub.in_degree(n) == 0]
        heads.extend(sorted(roots) if roots else [min(comp)])
    return heads


def _unit_cells(dag, th):
    """Rows split along R then L from every chain head, then columns along D then U (reference :505-654)."""
    for direction in ("R", "L", "D", "U"):
        for head in _heads(dag, direction):
            dag = _split_from_head(dag, head, direction, th)
    return dag


def line_from_head(dag, head, direction):
    """Nodes reachable from head along `direction` edges, breadth-first (reference utils/misc.py:430-448)."""
    out, queue = [], deque([head])
    while queue:
        u = queue.popleft()
        if u not in dag.nodes:
            continue
        out.append(u)
        queue.extend(v for v in dag.successors(u) if dag[u][v].get("dir") == direction)
    return out


def _grid_of(dag):
    """Row heads top to bottom x column heads left to right -> the node on both lines, or None (reference
    :657-695)."""
    rows = sorted(_heads(dag, "R"), key=lambda n: dag.nodes[n]["bbox"][1])
    cols = sorted(_heads(dag, "D"), key=lambda n: dag.nodes[n]["bbox"][0])
    col_sets = [set(line_from_head(dag, c, "D")) for c in cols]
    grid = []
    for r in rows:
        row_nodes = set(line_from_head(dag, r, "R"))
        grid.append([next(iter(row_nodes & cs)) if row_nodes & cs else None for cs in col_sets])
    return grid


def _place_cells(cells, grid):
    """row / col of a cell = its top-left grid position, spans = the rows / columns it covers (reference
    :613-646, 698-706)."""
    extent = {}
    for r, row in enumerate(grid):
        for c, cid in enumerate(row):
            if cid is None:
                continue
            e = extent.setdefault(cid, [r, r, c, c])
            e[0], e[1], e[2], e[3] = min(e[0], r), max(e[1], r), min(e[2], c), max(e[3], c)
    for cid, (r0, r1, c0, c1) in extent.items():
        cell = cells[cid]
        cell.row, cell.col, cell.row_span, cell.col_span = r0, c0, r1 - r0 + 1, c1 - c0 + 1


def _column_headers(grid, header_rows, cells, clustered_nodes):
    """Per column the distinct header-row cells top to bottom; headers of the region that head no column become
    cells (reference :722-758)."""
    used, col_headers = set(), []
    for c in range(len(grid[0])):
        ids = [grid[r][c] for r in range(len(grid)) if header_rows[r] and grid[r][c] is not None]
        used.update(ids)
        col_headers.append(sorted(set(ids), key=lambda h: cells[h].box[1]))
    region = {cell.id for group in clustered_nodes.values() for cell in group}
    for cell in cells.values():
        if cell.id not in used and cell.role == "header" and cell.id in region:
            cell.role = "cell"
    return col_headers


def _grid_box(grid, cells):
    boxes = [cells[cid].box for row in grid for cid in row if cid is not None]
    if not boxes:
        return (0.0, 0.0, 0.0, 0.0)
    return (min(b[0] for b in boxes), min(b[1] for b in boxes), max(b[2] for b in boxes), max(b[3] for b in boxes))


def parse_grid_from_bottom_up(cells, clustered_nodes, merge_same_column_values=False):
    """cells: id -> CellSchema of the table (row / col / spans and header roles are written in place);
    clustered_nodes: {"header", "cell", "empty", ...} -> cells of the region.  Returns (TableGridSchema, cells, graph)
    or None when no grid comes out (reference :874-923).  merge_same_column_values is not supported (the reference's
    TableSemanticParser never sets it)."""
    if merge_same_column_values:
        raise NotImplementedError("parse_grid_from_bottom_up: merge_same_column_values is not supported")
    members = clustered_nodes["cell"] + clustered_nodes["empty"] + clustered_nodes["header"]
    th = adjacency_thresholds([c.box for c in members])
    dag = _unit_cells(_grid_graph(clustered_nodes, th), th)
    grid = _grid_of(dag)
    if not grid or not grid[0]:
        return None
    header_rows = [all(cid is None or dag.nodes[cid]["role"] in ("header", "empty") for cid in row) for row in grid]
    grid = [[cid.split("__dup")[0] if cid is not None else None for cid in row] for row in grid]
    box = [int(v) for v in _grid_box(grid, cells)]
    _place_cells(cells, grid)
    col_headers = _column_headers(grid, header_rows, cells, clustered_nodes)
    return (TableGridSchema(id=None, n_row=len(grid), n_col=len(grid[0]), box=box, data=grid, col_headers=col_headers),
            cells, dag)
