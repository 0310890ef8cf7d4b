"""Host-side rules of the native library, checked on its sources (glim_b200/csrc/*.cu, *.cuh):

1. Every kernel launch goes through gb_launch: no triple-chevron launch anywhere else.
2. The launch counter (gb_ctx_kernel_launches) is written only by gb_launch, GB_CUB and the graph path of sweep_linearize.
3. Every cub device-wide call with temporary storage goes through GB_CUB (the size queries pass nullptr storage).
4. Every C-ABI entry point that takes a context, sweep, factor or peer slab enters through GB_ENTER (the context's lock and
   device), unless it is listed below with its reason; the lock and cudaSetDevice appear nowhere else but in GB_ENTER and
   the context lifetime and teardown functions.
5. align_up is called only by Carver: every block the host lays out is a Carver layout, run once to size and once to carve.
6. delete (of a handle) and cudaFree / cudaFreeHost appear only in the free and release functions listed below: each
   handle has one free function, which every destroy entry point and every failed creation calls.
7. gb_dev_malloc is called only by gb_dev_carve, and gb_dev_free only by the pool block's owner (gb_dev_block) and the free
   functions: every pool block is taken by one carve and held by one owner until a handle takes it over.
8. An asynchronous copy that may touch host memory (any cudaMemcpy*Async -- 1D, 2D, 3D, peer or symbol -- that is not
   explicitly cudaMemcpyDeviceToDevice) appears only in gb_upload, gb_download and gb_align_rounds, and in the functions
   listed below with their reasons: every other entry point moves its host arrays through the two helpers.  Every function
   that carves the context's pinned arena synchronises its stream in its own body (a stream synchronisation, gb_download or
   gb_align_rounds), or is listed with the callers that do, so no copy from the arena is pending when a call returns.

The function bodies are found by brace matching on the sources with comments, strings and preprocessor lines removed."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "glim_b200", "csrc")

HANDLE_PARAM = re.compile(r"\b(gb_ctx|gb_sweep|gb_factor|gb_peer_slab)\s*\*(?!\s*\*)")  # a handle taken, not a created one returned
# C-ABI entry points that take a handle but do not enter its context
NO_ENTER = {
    "gb_ctx_stream": "getter of a field fixed at creation",
    "gb_ctx_kernel_launches": "getter of the counter; no CUDA call",
    "gb_sweep_results_device": "getter of a pointer fixed at creation",
    "gb_sweep_stats": "getter of host fields",
    "gb_peer_slab_device_ptr": "getter: pointer arithmetic on the slab's own fields",
    "gb_vgicp_factor_create": "only retains the context (an atomic increment); no CUDA call",
    "gb_sweep_attach_slab": "host-only: records the caller's slab pointer",
    "gb_ctx_destroy": "teardown: locks the context itself, then releases it outside the lock",
    "gb_vgicp_factor_destroy": "teardown: sweep_free locks the context; the registry mutex guards the factor links",
    "gb_sweep_destroy": "teardown: sweep_free locks the context, then releases it outside the lock",
    "gb_peer_slab_destroy": "teardown: peer_slab_free locks the context, then releases it outside the lock",
}
# the only functions that may take the lock or set the device by hand: context lifetime, teardown, and calls on objects
# that keep no context (a device number only)
LOCK_OR_DEVICE_BY_HAND = {"ctx_create", "ctx_release", "gb_ctx_destroy", "sweep_free", "peer_slab_free", "gb_mem_info", "gb_cloud_destroy",
                          "gb_voxelmap_destroy", "gb_cloud_download", "gb_voxelmap_download"}
COUNTER_WRITERS = {"gb_launch", "sweep_linearize"}  # and the GB_CUB macro
# the only functions that may delete a handle or call cudaFree / cudaFreeHost
FREE_FUNCTIONS = {
    "cloud_free": "free function of gb_cloud",
    "voxelmap_free": "free function of gb_voxelmap",
    "sweep_free": "free function of gb_sweep",
    "peer_slab_free": "free function of gb_peer_slab",
    "ctx_release": "free function of gb_ctx (the last reference lets go)",
    "gb_vgicp_factor_destroy": "free function of gb_factor, which owns no device memory",
    "gb_dev_malloc": "the device pool gives its free blocks back to the driver when an allocation fails",
    "gb_dev_free": "the device pool frees a block it does not keep",
    "gb_arena_reserve": "the context's grow routine replaces its scratch / pinned buffer",
    "pool_block_free": "a sweep block evicted from the context's pool, or not kept by it",
    "dev_block_realloc": "a sweep's pair CSR block and a peer slab's pair list, replaced when a slab is attached",
}
XFER_HELPERS = {"gb_upload", "gb_download", "gb_align_rounds"}
# the only other functions that may copy between host and device asynchronously: each copies a pinned block of its own, or a
# layout of the context's pinned arena that the helpers' one copy per array cannot express
PINNED_COPIES = {
    "gb_sweep_create": "the sweep's own pinned descriptors and items",
    "gb_sweep_set_poses": "the sweep's own double-buffered pinned pose slots (no synchronisation)",
    "gb_sweep_fetch": "the sweep's own pinned results",
    "sweep_error": "the sweep's own pinned poses and results",
    "sweep_linearize": "the sweep's own pinned poses and results, captured into its graph",
    "sweep_learn_inliers": "the sweep's own pinned descriptors and items, re-uploaded when the items are re-sized",
    "sweep_follow_targets": "the sweep's own pinned descriptors, re-uploaded when a target changed",
    "gb_vgicp_align": "the align call's pinned block: states, offsets and poses written in place",
    "ct_upload": "the CT call block: descriptors and poses written in place, one copy",
    "ct_evaluate": "the CT call block's results",
    "gb_ct_gicp_align": "the CT call block's states",
    "gb_cloud_add_times": "the time table written in place in the pinned arena, one copy",
    "gb_peer_slab_fetch_async": "the peer slab's own pinned fetch block",
    "gb_overlap": "descriptors and poses adjacent in the pinned arena, one copy",
    "gb_region_growing": "a result-word tail: how many entries are used depends on the word the same copy brings back",
    "gb_min_cut": "a result-word tail: how many entries are used depends on the word the same copy brings back",
    "gb_gnc_align": "a result-word tail: how many entries are used depends on the word the same copy brings back",
    "gb_ransac_align": "per-block reads of the hypothesis counts into the pinned arena",
    "cloud_upload": "the fp64 -> fp32 pack writes the pinned planes directly, with threads",
}
# functions that carve ctx->pinned and leave the synchronisation to their callers
PINNED_SYNCED_BY_CALLER = {"ct_prepare": "the CT call block: ct_evaluate and gb_ct_gicp_align synchronise before they return"}


def strip_source(text):
    """Comments, string and character literals blanked (same length, newlines kept) and preprocessor lines split off:
    returns (code, [preprocessor directives with their continuation lines joined])."""
    out = []
    i, n = 0, len(text)
    while i < n:
        c = text[i]
        if text.startswith("//", i):
            j = text.find("\n", i)
            j = n if j < 0 else j
            out.append(" " * (j - i))
            i = j
        elif text.startswith("/*", i):
            j = text.find("*/", i + 2)
            j = n if j < 0 else j + 2
            out.append(re.sub(r"[^\n]", " ", text[i:j]))
            i = j
        elif c in "\"'":
            j = i + 1
            while j < n and text[j] != c:
                j += 2 if text[j] == "\\" else 1
            out.append(c + " " * (j - i - 1) + c)
            i = j + 1
        else:
            out.append(c)
            i += 1
    code = "".join(out)
    lines = code.split("\n")
    directives, k = [], 0
    while k < len(lines):
        if lines[k].lstrip().startswith("#"):
            start = k
            while lines[k].rstrip().endswith("\\") and k + 1 < len(lines):
                k += 1
            directives.append("\n".join(lines[start:k + 1]))
            for m in range(start, k + 1):
                lines[m] = " " * len(lines[m])
        k += 1
    return "\n".join(lines), directives


def match_brace(code, i):
    depth = 0
    for j in range(i, len(code)):
        if code[j] == "{":
            depth += 1
        elif code[j] == "}":
            depth -= 1
            if depth == 0:
                return j
    raise ValueError("unbalanced braces")


def function_name(header):
    """Name of the function a block header defines (the identifier before its last parenthesised group), else None."""
    h = re.sub(r"\b(const|noexcept|override)\s*$", "", header.rstrip()).rstrip()
    if not h.endswith(")"):
        return None
    depth = 0
    for j in range(len(h) - 1, -1, -1):
        depth += h[j] == ")"
        depth -= h[j] == "("
        if depth == 0:
            m = re.search(r"([A-Za-z_]\w*)\s*(<[^()]*>)?\s*$", h[:j])
            return m.group(1) if m else None
    return None


def functions(code):
    """[(name, header, body_start, body_end)] of the function definitions outside other functions (namespaces are transparent)."""
    found, seg, i = [], 0, 0
    while i < len(code):
        c = code[i]
        if c == "{":
            header = code[seg:i]
            if re.search(r"\bnamespace\b[\w\s]*$", header):
                seg = i = i + 1
                continue
            end = match_brace(code, i)
            name = function_name(header)
            if name:
                found.append((name, header, i, end))
            seg = i = end + 1
            continue
        if c in ";}":
            seg = i + 1
        i += 1
    return found


def sources(csrc):
    out = []
    for f in sorted(os.listdir(csrc)):
        if f.endswith((".cu", ".cuh")):
            code, directives = strip_source(open(os.path.join(csrc, f)).read())
            out.append((f, code, directives, functions(code)))
    return out


def enclosing(funcs, pos):
    for name, _, b, e in funcs:
        if b <= pos <= e:
            return name
    return None


def line_of(code, pos):
    return code.count("\n", 0, pos) + 1


def struct_body(code, name):
    """(start, end) of the body of struct `name` in code, or None."""
    m = re.search(r"\bstruct\s+" + name + r"\s*\{", code)
    return (m.end() - 1, match_brace(code, m.end() - 1)) if m else None


def pool_uses(code, funcs):
    """[(pos, 'malloc' | 'free', allowed)] of every use of gb_dev_malloc / gb_dev_free other than their declarations and
    definitions (rule 7)."""
    owner = struct_body(code, "gb_dev_block")
    out = []
    for m in re.finditer(r"\bgb_dev_(malloc|free)\b", code):
        if re.search(r"\b(cudaError_t|void)\s+$", code[max(0, m.start() - 40):m.start()]):
            continue
        if m.group(1) == "malloc":
            allowed = enclosing(funcs, m.start()) == "gb_dev_carve"
        else:
            allowed = enclosing(funcs, m.start()) in FREE_FUNCTIONS or bool(owner and owner[0] < m.start() < owner[1])
        out.append((m.start(), m.group(1), allowed))
    return out


def host_copies(code, funcs):
    """[(pos, enclosing function)] of every asynchronous copy that may touch host memory (rule 8)."""
    out = []
    for m in re.finditer(r"\bcudaMemcpy\w*Async\s*\(", code):
        if not re.search(r"\bcudaMemcpyDeviceToDevice\b", code[m.end():code.find(";", m.end())]):
            out.append((m.start(), enclosing(funcs, m.start())))
    return out


def pinned_carvers(code, funcs):
    """[(pos, function, synchronises in its body)] of every carve of a context's pinned arena (rule 8)."""
    out = []
    for m in re.finditer(r"\bgb_carve\s*\([^,;]+,\s*[\w.>-]*\bpinned\b", code):
        name = enclosing(funcs, m.start())
        b, e = next((b, e) for n, _, b, e in funcs if n == name)
        out.append((m.start(), name, bool(re.search(r"\bcudaStreamSynchronize\s*\(|\bgb_download\s*\(|\bgb_align_rounds\s*\(", code[b:e]))))
    return out


def violations(csrc):
    """{rule: [offending site]} for rules 1-8 of this module's docstring."""
    bad = {1: [], 2: [], 3: [], 4: [], 5: [], 6: [], 7: [], 8: []}
    enters = 0
    for f, code, directives, funcs in sources(csrc):
        where = lambda pos: f"{f}:{line_of(code, pos)} ({enclosing(funcs, pos)})"
        bad[7] += [where(pos) for pos, _, allowed in pool_uses(code, funcs) if not allowed]
        bad[7] += [f"{f}: {d.splitlines()[0].strip()}" for d in directives if re.search(r"\bgb_dev_(malloc|free)\b", d)]
        bad[8] += [where(pos) for pos, name in host_copies(code, funcs) if name not in XFER_HELPERS and name not in PINNED_COPIES]
        bad[8] += [f"{f}: {d.splitlines()[0].strip()}" for d in directives if re.search(r"\bcudaMemcpy\w*Async\b", d)]
        bad[8] += [where(pos) + " carves the pinned arena and does not synchronise" for pos, name, syncs in pinned_carvers(code, funcs)
                   if not syncs and name not in PINNED_SYNCED_BY_CALLER]
        carver = struct_body(code, "Carver")
        for m in re.finditer(r"\balign_up\b", code):
            definition = re.search(r"\bsize_t\s+$", code[max(0, m.start() - 40):m.start()])
            if not (definition or (carver and carver[0] < m.start() < carver[1])):
                bad[5].append(where(m.start()))
        for m in re.finditer(r"\bdelete\b|\bcudaFree(Host)?\s*\(", code):
            if enclosing(funcs, m.start()) not in FREE_FUNCTIONS:
                bad[6].append(where(m.start()))
        for d in directives:
            if re.search(r"\balign_up\b|\bdelete\b|\bcudaFree", d):
                bad[5 if "align_up" in d else 6].append(f"{f}: {d.splitlines()[0].strip()}")
        for m in re.finditer(r"<<<", code):
            if enclosing(funcs, m.start()) != "gb_launch":
                bad[1].append(where(m.start()))
        for m in re.finditer(r"(->|\.)\s*launches\s*(\+\+|--|[-+]?=(?!=))|(\+\+|--)\s*[\w()]+\s*->\s*launches\b", code):
            if enclosing(funcs, m.start()) not in COUNTER_WRITERS:
                bad[2].append(where(m.start()))
        for d in directives:
            if re.search(r"\blaunches\b", d) and not re.match(r"\s*#\s*define\s+GB_CUB\(", d):
                bad[2].append(f"{f}: {d.splitlines()[0].strip()}")
            if re.search(r"\bGB_LOCK\s*\(|\bcudaSetDevice\s*\(", d) and not re.match(r"\s*#\s*define\s+(GB_ENTER|GB_LOCK)\(", d):
                bad[4].append(f"{f}: {d.splitlines()[0].strip()}")
        for m in re.finditer(r"\bcub\s*::\s*Device\w+\s*::\s*\w+", code):
            through_wrapper = re.search(r"\bGB_CUB\s*\(\s*[^,;]+,\s*$", code[max(0, m.start() - 200):m.start()])
            size_query = re.match(r"\s*\(\s*nullptr\s*,", code[m.end():])
            if not (through_wrapper or size_query):
                bad[3].append(where(m.start()))
        for name, header, b, e in funcs:
            if not re.match(r"\s*extern\s*\"\s*\"", header):
                continue
            params = header[header.index(name) + len(name):]
            if not HANDLE_PARAM.search(params):
                continue
            if "GB_ENTER(" in code[b:e]:
                enters += 1
            elif name not in NO_ENTER:
                bad[4].append(f"{f}: {name} does not enter through GB_ENTER")
        for m in re.finditer(r"\bGB_LOCK\s*\(|\bcudaSetDevice\s*\(", code):
            if enclosing(funcs, m.start()) not in LOCK_OR_DEVICE_BY_HAND:
                bad[4].append(where(m.start()))
    return bad, enters


def parsed_inventory(csrc):
    """Sanity numbers of the parse, so that a rule cannot pass because the parser found nothing."""
    names, launches_in_helper, cub_calls, carver_align, frees = set(), 0, 0, 0, 0
    pool = {"malloc": 0, "free": 0}  # allowed uses of gb_dev_malloc / gb_dev_free (rule 7)
    xfer = {"gb_upload": 0, "gb_download": 0, "copies": {}, "carvers": set()}  # the helpers' uses, the copies, the pinned carves (rule 8)
    for f, code, _, funcs in sources(csrc):
        names.update(n for n, *_ in funcs)
        launches_in_helper += sum(1 for m in re.finditer(r"<<<", code) if enclosing(funcs, m.start()) == "gb_launch")
        cub_calls += len(re.findall(r"\bGB_CUB\s*\(", code))
        carver = struct_body(code, "Carver")
        if carver:
            carver_align += len(re.findall(r"\balign_up\s*\(", code[carver[0]:carver[1]]))
        frees += sum(1 for m in re.finditer(r"\bdelete\b|\bcudaFree(Host)?\s*\(", code) if enclosing(funcs, m.start()) in FREE_FUNCTIONS)
        for _, kind, allowed in pool_uses(code, funcs):
            pool[kind] += allowed
        for m in re.finditer(r"\b(gb_upload|gb_download)\s*\(", code):
            if enclosing(funcs, m.start()) not in (None, m.group(1)):  # a call, not the declaration or the definition
                xfer[m.group(1)] += 1
        for _, name in host_copies(code, funcs):
            xfer["copies"][name] = xfer["copies"].get(name, 0) + 1
        xfer["carvers"] |= {name for _, name, _ in pinned_carvers(code, funcs)}
    return names, launches_in_helper, cub_calls, carver_align, frees, pool, xfer


def test_parser_sees_the_library():
    names, launches_in_helper, cub_calls, carver_align, frees, pool, xfer = parsed_inventory(CSRC)
    assert {"gb_launch", "sweep_linearize", "gb_preprocess", "gb_vgicp_align", "gb_deskew", "knn_device", "table_build", "gb_dev_carve"} <= names
    assert set(FREE_FUNCTIONS) <= names
    assert launches_in_helper == 1
    assert cub_calls >= 10
    assert carver_align == 1
    assert frees >= len(FREE_FUNCTIONS)
    # the carve's one allocation; the owner's free and those of cloud_free (3 blocks) and voxelmap_free (2)
    assert pool == {"malloc": 1, "free": 6}
    # the helpers' calls; each listed site still copies, and each helper copies in one place
    assert xfer["gb_upload"] >= 9 and xfer["gb_download"] >= 17
    assert set(PINNED_COPIES) <= set(xfer["copies"])
    assert all(xfer["copies"].get(h) == 1 for h in XFER_HELPERS)
    assert set(PINNED_SYNCED_BY_CALLER) <= xfer["carvers"] and len(xfer["carvers"]) >= 8
    _, enters = violations(CSRC)
    assert enters >= 29  # gb_peer_slab_destroy is teardown now: peer_slab_free locks the context by hand


def test_every_kernel_launch_goes_through_gb_launch():
    assert violations(CSRC)[0][1] == []


def test_launch_counter_written_only_by_the_helpers_and_the_graph_path():
    assert violations(CSRC)[0][2] == []


def test_every_cub_call_goes_through_gb_cub():
    assert violations(CSRC)[0][3] == []


def test_every_context_bound_entry_point_enters_its_context():
    assert violations(CSRC)[0][4] == []


def test_align_up_only_in_carver():
    assert violations(CSRC)[0][5] == []


def test_handles_freed_only_by_their_free_functions():
    assert violations(CSRC)[0][6] == []


def test_pool_blocks_taken_by_one_carve_and_returned_by_one_owner():
    assert violations(CSRC)[0][7] == []


def test_host_transfers_go_through_the_two_helpers():
    assert violations(CSRC)[0][8] == []
