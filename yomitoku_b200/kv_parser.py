"""Key-value items of a table: `parse_kv_items` (reference src/yomitoku/kv_parser.py:1-626).

Cells and headers are assigned to the model's kv_item regions; inside a region headers point at the cells and headers
next to them (R / D edges).  Per connected part of that graph every root header is walked depth-first along R and
along D, and the direction that reaches more values wins: each value reached becomes a KvItem whose key is the header
path.  Headers and cells outside every region are then rescued by three fallbacks, and cells still without a key
become key-less items.  Host code like in the reference.

One deliberate difference: the reference walks the root headers of a part in the iteration order of a Python set of
cell ids, which follows the per-process string hash, so the order of items whose values share a top edge changes from
run to run.  Here the roots are walked in the order the graph holds them (headers in cell order).
"""
import networkx as nx

from .document_analyzer import is_bottom_adjacent, is_contained, is_right_adjacent, overlap_ratio
from .schemas import KvItemSchema

__all__ = ["parse_kv_items"]

NESTED_TH = 0.8      # share of an interval inside another that makes it nested (reference :12-13)


def _overlap_len(i1, i2, j1, j2):
    return max(0.0, min(i2, j2) - max(i1, j1))


def _nested(parent_lo, parent_hi, lo, hi):
    """Share of [lo, hi] inside [parent_lo, parent_hi] (reference :308-313)."""
    return _overlap_len(parent_lo, parent_hi, lo, hi) / (hi - lo) if hi - lo > 0 else 0.0


def _hull(a, b):
    return [min(a[0], b[0]), min(a[1], b[1]), max(a[2], b[2]), max(a[3], b[3])]


def _regions_of(nodes, regions):
    """cell / empty -> the region covering most of it (> 20 % inside, first on ties); header -> every region it is
    > 20 % inside (reference :16-56)."""
    cell_region, header_regions = {}, {}
    if not regions:
        return cell_region, header_regions
    for cell in nodes["cell"] + nodes["empty"]:
        best, best_ratio = None, 0.0
        for region in regions:
            if is_contained(region.box, cell.box, threshold=0.2):
                ratio = overlap_ratio(cell.box, region.box)[0]
                if ratio > best_ratio:
                    best, best_ratio = region.id, ratio
        if best is not None:
            cell_region[cell.id] = best
    for header in nodes["header"]:
        regs = {r.id for r in regions if is_contained(r.box, header.box, threshold=0.2)}
        if regs:
            header_regions[header.id] = regs
    return cell_region, header_regions


def _adopt_orphan_headers(headers, header_regions):
    """A header in no region takes the regions of every region header right of it, repeated until nothing changes
    (chains of orphans; reference :59-108)."""
    orphans = {h.id for h in headers if not header_regions.get(h.id)}
    changed = True
    while changed:
        changed = False
        for orphan in headers:
            if orphan.id not in orphans:
                continue
            regs = set(header_regions.get(orphan.id, set()))
            for other in headers:
                if other.id != orphan.id and header_regions.get(other.id) and is_right_adjacent(orphan.box, other.box):
                    regs |= header_regions[other.id]
            if regs and regs != header_regions.get(orphan.id):
                header_regions[orphan.id] = regs
                changed = True
    return header_regions


def _link(dag, a, b):
    """Edges from a to b (R / D) and back (L / U) where b is right of / below a."""
    if is_right_adjacent(a.box, b.box):
        dag.add_edge(a.id, b.id, dir="R")
        dag.add_edge(b.id, a.id, dir="L")
    if is_bottom_adjacent(a.box, b.box):
        dag.add_edge(a.id, b.id, dir="D")
        dag.add_edge(b.id, a.id, dir="U")


def _kv_graph(nodes, regions):
    """The adjacency graph inside the regions (reference :111-244): header -> cell, header -> empty, header -> header
    sharing a region, cell -> cell of one region."""
    cell_region, header_regions = _regions_of(nodes, regions)
    header_regions = _adopt_orphan_headers(nodes["header"], header_regions)
    dag = nx.DiGraph()
    for n in nodes["header"] + nodes["cell"] + nodes["empty"]:
        dag.add_node(n.id, id=n.id, bbox=n.box, role=n.role, contents=n.contents)
    for values in (nodes["cell"], nodes["empty"]):
        for header in nodes["header"]:
            regs = header_regions.get(header.id)
            if not regs:
                continue
            for cell in values:
                if cell_region.get(cell.id) in regs:
                    _link(dag, header, cell)
    for node in nodes["header"]:
        for parent in nodes["header"]:
            if node.id == parent.id:
                continue
            pr, nr = header_regions.get(parent.id), header_regions.get(node.id)
            if pr and nr and pr & nr:
                _link(dag, parent, node)
    for node in nodes["cell"]:
        nr = cell_region.get(node.id)
        if nr is None:
            continue
        for parent in nodes["cell"]:
            if node.id != parent.id and cell_region.get(parent.id) == nr:
                _link(dag, parent, node)
    return dag, cell_region, header_regions


def _roots(dag, direction, order, part):
    """Headers of the set `part` (in the order of the list `order`) without a `direction` edge from another header of
    it (reference :256-277)."""
    roots = []
    for h in order:
        if dag.nodes[h]["role"] != "header":
            continue
        if not any(u in part and dag.nodes[u]["role"] == "header" and dag[u][h].get("dir") == direction
                   for u in dag.predecessors(h)):
            roots.append(h)
    return roots


def _walk(dag, node_id, path, items, cells, used, direction):
    """Depth-first from a header along `direction`; a value reached becomes an item keyed by the path (reference
    :280-305)."""
    if dag.nodes[node_id]["role"] in ("cell", "empty"):
        box = _hull(cells[node_id].box, cells[path[0]].box) if path else cells[node_id].box
        items.append(KvItemSchema(id=None, key=list(path), value=node_id, box=box))
        used[node_id] = cells[node_id]
        for k in path:
            used[k] = cells[k]
        return
    path = path + [node_id]
    for v in dag.successors(node_id):
        if v not in path and dag[node_id][v].get("dir") == direction:
            _walk(dag, v, path, items, cells, used, direction)


def _rescue_nested_orphans(orphans, items, cells, used):
    """An orphan header that holds key heads nested in it - to its right inside its rows, or below it in a chain of
    narrower headers inside its columns - is put in front of their keys (reference :316-392)."""
    for orphan in orphans:
        ox1, oy1, ox2, oy2 = orphan.box
        ow, oh = ox2 - ox1, oy2 - oy1
        heads = {}
        for kv in items:
            if kv.key:
                head = cells.get(kv.key[0])
                if head is not None and head.id != orphan.id:
                    heads[head.id] = head
        targets = {h.id for h in heads.values()
                   if h.box[0] >= ox2 - ow * 0.1 and (h.box[3] - h.box[1]) < oh * 0.9
                   and _nested(oy1, oy2, h.box[1], h.box[3]) >= NESTED_TH}
        below = {h.id: h for h in heads.values()
                 if (h.box[2] - h.box[0]) < ow * 0.9 and _nested(ox1, ox2, h.box[0], h.box[2]) >= NESTED_TH}
        frontier = [h for h in below.values() if is_bottom_adjacent(orphan.box, h.box)]
        linked = {h.id for h in frontier}
        while frontier:
            cur = frontier.pop()
            for h in below.values():
                if h.id not in linked and is_bottom_adjacent(cur.box, h.box):
                    linked.add(h.id)
                    frontier.append(h)
        targets |= linked
        if not targets:
            continue
        for kv in items:
            if kv.key and kv.key[0] in targets:
                kv.key = [orphan.id] + list(kv.key)
                kv.box = _hull(kv.box, orphan.box) if kv.box else list(orphan.box)
        used[orphan.id] = cells[orphan.id]


def _rescue_orphan_chains(orphans, orphan_cells, items, cells, used):
    """From each orphan header, chains of orphan cells to its right and below it: the last cell of a chain is the
    value, the cells on the way are keys after the header (reference :395-454)."""
    paired, as_keys = set(), set()
    for orphan in orphans:
        for adjacent in (is_right_adjacent, is_bottom_adjacent):
            seen = set()

            def chain(node, path):
                children = [c for c in orphan_cells if c.id not in seen and c.id not in paired
                            and c.id not in as_keys and adjacent(node.box, c.box)]
                if not children:
                    if node.id == orphan.id:
                        return
                    items.append(KvItemSchema(id=None, key=list(path), value=node.id,
                                              box=_hull(cells[path[0]].box, node.box)))
                    for k in path:
                        used[k] = cells[k]
                    used[node.id] = cells[node.id]
                    paired.add(node.id)
                    as_keys.update(path[1:])
                    return
                seen.update(c.id for c in children)
                for c in children:
                    chain(c, path + [node.id])

            chain(orphan, [])
    return paired, as_keys


def _rescue_continuations(items, candidates, cells, used):
    """A key-less cell right of (first) or below a keyed value, with the same row height / column width (both
    intervals >= 80 % inside each other), inherits that value's key; repeated so that runs of such cells chain
    (reference :457-536)."""
    inherited = set()
    value_key = {kv.value: list(kv.key) for kv in items if kv.key}
    directions = ((is_right_adjacent, (1, 3)), (is_bottom_adjacent, (0, 2)))
    remaining = {c.id: c for c in candidates}
    changed = True
    while changed:
        changed = False
        for cell in list(remaining.values()):
            key = None
            for adjacent, (lo, hi) in directions:
                for vid, vkey in value_key.items():
                    vc = cells.get(vid)
                    if vc is None or not adjacent(vc.box, cell.box):
                        continue
                    if (_nested(vc.box[lo], vc.box[hi], cell.box[lo], cell.box[hi]) < NESTED_TH
                            or _nested(cell.box[lo], cell.box[hi], vc.box[lo], vc.box[hi]) < NESTED_TH):
                        continue
                    key = vkey
                    break
                if key is not None:
                    break
            if key is None:
                continue
            items.append(KvItemSchema(id=None, key=list(key), value=cell.id, box=_hull(cells[key[0]].box, cell.box)))
            used[cell.id] = cells[cell.id]
            for k in key:
                used[k] = cells[k]
            value_key[cell.id] = list(key)
            inherited.add(cell.id)
            del remaining[cell.id]
            changed = True
    return inherited


def parse_kv_items(nodes, cells, regions):
    """nodes: {"header", "cell", "empty", ...} -> cells; cells: id -> CellSchema; regions: the kv_item RegionSchemas
    (ids set).  Returns (items, graph, id -> cells the items use) (reference :539-626)."""
    dag, cell_region, header_regions = _kv_graph(nodes, regions)
    items, used = [], {}
    for comp in nx.weakly_connected_components(dag):
        part = [n for n in dag.nodes if n in comp]
        found = {}
        for direction in ("R", "D"):
            its, us = [], {}
            for root in _roots(dag, direction, part, comp):
                _walk(dag, root, [], its, cells, us, direction)
            found[direction] = (its, us)
        h_items, h_used = found["R"]
        v_items, v_used = found["D"]
        if len({kv.value for kv in v_items}) > len({kv.value for kv in h_items}):
            items.extend(v_items)
            used.update(v_used)
            drop = ("R", "L")
        else:
            items.extend(h_items)
            used.update(h_used)
            drop = ("D", "U")
        dag.remove_edges_from([(u, v) for u, v, d in dag.edges(part, data=True) if v in comp and d.get("dir") in drop])
    orphans = sorted((h for h in nodes["header"] if not header_regions.get(h.id)), key=lambda h: (h.box[1], h.box[0]))
    _rescue_nested_orphans(orphans, items, cells, used)
    visited = {kv.value for kv in items}
    orphan_cells = [c for c in nodes["cell"] + nodes["empty"] if c.id not in cell_region and c.id not in visited]
    paired, as_keys = _rescue_orphan_chains(orphans, orphan_cells, items, cells, used)
    visited |= paired | as_keys
    unkeyed = [c for c in nodes["cell"] + nodes["empty"] if c.id not in visited]
    visited |= _rescue_continuations(items, unkeyed, cells, used)
    for cell in nodes["cell"] + nodes["empty"]:
        if cell.id not in visited:
            items.append(KvItemSchema(id=None, key=[], value=cell.id, box=cell.box))
            used[cell.id] = cells[cell.id]
    return items, dag, used
