"""The smart and Frappe feature stages on the GPU: deep_ctr/Feature_pipeline/get_smart_feature.py (a 128-column CSV ->
libsvm through a feature_map file, plus its get_feature_map builder) and get_frape_feature.py (the Frappe label
rewrite), through the ctr_smart_* / ctr_frappe_* entry points (csrc/smart_feature.cu).

Inputs are read in pieces of whole lines and uploaded one at a time, so they may be larger than device memory; only the
feature_map text and its table (48 bytes a slot) stay resident, plus the builder's table (16 bytes a slot) and key
arena while it runs.  The libsvm files are byte-identical to what the reference writes under Python 2.7 wherever its
result is defined.  Deliberate deviations (DESIGN.md §2.12), none of which changes such bytes:
  * inputs are taken in sorted path order (glob order in the reference);
  * where the reference's concurrent workers would write one file (several `va` / `te` inputs) the inputs are
    concatenated in that order; inputs whose output names collide raise before anything is written;
  * a `tr` path with fewer than four '_' pieces raises before anything is written (the reference's IndexError kills
    its pool after partial writes);
  * the feature_map the builder writes is in fid order (Python 2 dict order there); compare it as a set of lines."""
from __future__ import annotations

import glob
import os
from typing import Dict, List, Tuple

import torch

from . import _lib
from ._lib import check
from .ops import _stream
from .text_chunks import Timer, pieces, scratch, upload

_L = _lib.raw()

# the file format: 28 named columns, then xgbf_0 .. xgbf_99; continuous = 11..27, categorical = 1..10 and 28..127
NAMED = (b"is_click", b"u_pl", b"u_ppvn", b"u_de", b"u_os", b"u_t", b"a_m_w", b"a_b_w", b"c_h", b"c_w", b"c_al",
         b"u_ctr", b"a_a_ctr", b"a_t_ctr", b"c_q_ctr", b"c_al_ctr", b"c_n_ctr", b"c_t_ctr", b"c_t_n_ctr",
         b"u_a_city_ctr", b"u_a_age_ctr", b"u_a_x_ctr", b"u_a_g_ctr", b"u_a_c_ctr", b"c_q_a_ctr", b"c_q_t_sim",
         b"c_q_adtype_ctr", b"c_mw_a_ctr")
CSV_COLUMNS = NAMED + tuple(b"xgbf_%d" % i for i in range(100))
PATTERNS = {"tr": "/*part*", "va": "/*verify", "te": "/*test"}


class SmartFeatureError(ValueError):
    pass


def input_files(input_dir: str, task_type: str) -> List[str]:
    """glob(input_dir + pattern) of the task (:124-131), in sorted order."""
    if task_type not in PATTERNS:
        raise SmartFeatureError(f"task_type must be one of tr, va, te (got {task_type!r})")
    return sorted(glob.glob(input_dir + PATTERNS[task_type]))


def smart_outputs(files: List[str], output_dir: str, task_type: str) -> List[Tuple[str, List[str]]]:
    """(output path, its inputs) in order (:64-67): tr writes output_dir + 'tr_' + path.rsplit('_')[3] + '.libsvm' per
    input, va / te write every input to one file.  Raises where the reference's names are not usable."""
    if task_type != "tr":
        return [(output_dir + task_type + ".libsvm", list(files))] if files else []
    outs = []
    for path in files:
        parts = path.rsplit("_")
        if len(parts) < 4:
            raise SmartFeatureError(f"{path}: fewer than 4 '_'-separated pieces, so the reference's "
                                    "path.rsplit('_')[3] raises IndexError (nothing was written)")
        outs.append((output_dir + "tr_" + parts[3] + ".libsvm", [path]))
    return _no_collisions(outs)


def frappe_outputs(input_dir: str) -> List[Tuple[str, List[str]]]:
    """(path.split('.')[0] + '_.libsvm', [path]) for each glob(input_dir + '/*libsvm') in sorted order (:17, :58)."""
    return _no_collisions([(p.split(".")[0] + "_.libsvm", [p]) for p in sorted(glob.glob(input_dir + "/*libsvm"))])


def _no_collisions(outs):
    seen = {}
    for out, ins in outs:
        if out in seen:
            raise SmartFeatureError(f"{seen[out]} and {ins[0]} both write {out} (the reference's workers would "
                                    "overwrite each other; nothing was written)")
        seen[out] = ins[0]
    return outs


def _device(device):
    dev = torch.device(device)
    if dev.type != "cuda":
        raise _lib.CtrError("smart_feature runs on a CUDA device (there is no CPU path)")
    return dev


def _check_sizes(chunk_bytes, *caps):
    if not (1 <= chunk_bytes < (1 << 30)) or not all(1 <= c <= (1 << 31) for c in caps):
        raise ValueError("chunk_bytes must be in [1, 2^30) and every capacity in [1, 2^31]")


def _stream_lines(paths, fh, dev, chunk_bytes, timer, ws_fn, plan_fn, write_fn) -> Tuple[int, int]:
    """every piece of every path through plan / write, appended to fh; -> (lines read, lines written)"""
    info = torch.empty(3, dtype=torch.int64, device=dev)
    n_in = n_out = 0
    for path in paths:
        for data in pieces(path, chunk_bytes):
            text = upload(data, dev)
            ws_bytes = int(ws_fn(len(data)))
            ws = scratch(ws_bytes, dev)
            timer.start()
            plan_fn(text.data_ptr(), len(data), info.data_ptr(), ws.data_ptr(), ws_bytes)
            timer.stop()
            lines, kept, nbytes = info.tolist()
            out = scratch(nbytes, dev)
            timer.start()
            write_fn(text.data_ptr(), len(data), out.data_ptr(), ws.data_ptr(), ws_bytes)
            timer.stop()
            fh.write(out[:nbytes].cpu().numpy().tobytes())
            n_in += lines
            n_out += kept
    return n_in, n_out


def build_feature_map(files: List[str], dev, chunk_bytes: int, capacity: int, arena_bytes: int, timer: Timer) -> bytes:
    """get_feature_map (:27-53, with CSV_COLUMNS[i] at :32 read as fname) over files in order -> the feature_map text
    in fid order: name|UNK for the 128 names (fids 1..128), then each new key in order of its first (line, column)."""
    table = torch.zeros(int(_L.ctr_smart_build_table_bytes(capacity)), dtype=torch.uint8, device=dev)
    state = torch.zeros(19, dtype=torch.int64, device=dev)
    arena = scratch(arena_bytes, dev)
    info = torch.empty(2, dtype=torch.int64, device=dev)
    line_base = 0
    for path in files:
        for data in pieces(path, chunk_bytes):
            text = upload(data, dev)
            ws_bytes = int(_L.ctr_smart_build_insert_workspace_bytes(len(data)))
            ws = scratch(ws_bytes, dev)
            timer.start()
            check(_L.ctr_smart_build_insert(text.data_ptr(), len(data), line_base, table.data_ptr(), capacity,
                                            arena.data_ptr(), arena_bytes, state.data_ptr(), info.data_ptr(),
                                            ws.data_ptr(), ws_bytes, _stream()), "ctr_smart_build_insert")
            timer.stop()
            n, dropped = info.tolist()
            full = int(state[1])
            if dropped or full:
                raise SmartFeatureError(
                    f"{path}: the feature_map builder's " + (
                        f"key table is full (build_capacity={capacity} slots; {dropped} keys found no slot): raise "
                        "build_capacity (about twice the number of distinct keys)" if dropped else
                        f"key arena is full (build_arena_bytes={arena_bytes}): raise build_arena_bytes (the bytes of "
                        "every distinct categorical value, plus one each)") + " (nothing was written)")
            line_base += n
    ws_bytes = int(_L.ctr_smart_build_workspace_bytes(capacity))
    ws = scratch(ws_bytes, dev)
    timer.start()
    check(_L.ctr_smart_build_finish(table.data_ptr(), capacity, arena.data_ptr(), state.data_ptr(), info.data_ptr(),
                                    ws.data_ptr(), ws_bytes, _stream()), "ctr_smart_build_finish")
    timer.stop()
    _, nbytes = info.tolist()
    out = scratch(nbytes, dev)
    timer.start()
    check(_L.ctr_smart_build_render(table.data_ptr(), capacity, arena.data_ptr(), out.data_ptr(), ws.data_ptr(),
                                    ws_bytes, _stream()), "ctr_smart_build_render")
    timer.stop()
    seeded = b"".join(b"%s|UNK %d\n" % (name, i + 1) for i, name in enumerate(CSV_COLUMNS))
    return seeded + out[:nbytes].cpu().numpy().tobytes()


def smart_feature(input_dir: str, output_dir: str, task_type: str = "tr", build_feature_map_first: bool = False,
                  device="cuda", chunk_bytes: int = 64 << 20, table_capacity: int = None,
                  build_capacity: int = 1 << 24, build_arena_bytes: int = 256 << 20) -> Dict:
    """get_smart_feature.py's main for one task_type: reads output_dir + 'feature_map' (plain string concatenation,
    as the reference builds its paths) and writes the libsvm files of smart_outputs().  build_feature_map_first runs
    the builder over the `tr` inputs and writes that feature_map before (the reference's commented-out call, :127).
    table_capacity = slots of the map table (default: twice the map's lines); it raises when too small, before
    anything is written.  Returns the outputs, line counts and the device milliseconds of each pass."""
    dev = _device(device)
    files = input_files(input_dir, task_type)
    outs = smart_outputs(files, output_dir, task_type)
    with torch.cuda.device(dev):
        return _smart(input_dir, output_dir, outs, build_feature_map_first, dev, int(chunk_bytes), table_capacity,
                      int(build_capacity), int(build_arena_bytes))


def _smart(input_dir, output_dir, outs, build, dev, chunk_bytes, table_capacity, build_capacity, arena_bytes):
    timers = {k: Timer() for k in ("build", "map", "emit")}
    map_path = output_dir + "feature_map"
    if build:
        _check_sizes(chunk_bytes, build_capacity, arena_bytes)
        text = build_feature_map(input_files(input_dir, "tr"), dev, chunk_bytes, build_capacity, arena_bytes,
                                 timers["build"])
        with open(map_path, "wb") as fh:
            fh.write(text)
    with open(map_path, "rb") as fh:                   # a missing feature_map raises here, before any output
        map_bytes = fh.read()
    cap = int(table_capacity) if table_capacity else max(2 * (map_bytes.count(b"\n") + 1), 1024)
    _check_sizes(chunk_bytes, cap)
    map_text = upload(map_bytes, dev)
    table = torch.zeros(int(_L.ctr_smart_map_table_bytes(cap)), dtype=torch.uint8, device=dev)
    col_fid = torch.empty(256, dtype=torch.int64, device=dev)
    info = torch.empty(3, dtype=torch.int64, device=dev)
    ws_bytes = int(_L.ctr_smart_map_workspace_bytes(len(map_bytes)))
    ws = scratch(ws_bytes, dev)
    map_ptr = map_text.data_ptr() if map_bytes else None
    timers["map"].start()
    check(_L.ctr_smart_map_build(map_ptr, len(map_bytes), table.data_ptr(), cap, col_fid.data_ptr(), info.data_ptr(),
                                 ws.data_ptr(), ws_bytes, _stream()), "ctr_smart_map_build")
    timers["map"].stop()
    del ws
    map_lines, keys, dropped = info.tolist()
    if dropped:
        raise SmartFeatureError(f"{map_path}: the feature_map table is full (table_capacity={cap} slots; {dropped} "
                                "keys found no slot): raise table_capacity (about twice the map's lines; nothing was "
                                "written)")

    common = (map_ptr, table.data_ptr(), cap, col_fid.data_ptr())

    def plan(text, n, info_ptr, ws_ptr, ws_bytes):
        check(_L.ctr_smart_emit_plan(text, n, *common, info_ptr, ws_ptr, ws_bytes, _stream()), "ctr_smart_emit_plan")

    def write(text, n, out, ws_ptr, ws_bytes):
        check(_L.ctr_smart_emit_write(text, n, *common, out, ws_ptr, ws_bytes, _stream()), "ctr_smart_emit_write")

    lines = {}
    for out, ins in outs:
        with open(out, "wb") as fh:
            lines[out] = _stream_lines(ins, fh, dev, chunk_bytes, timers["emit"], _L.ctr_smart_emit_workspace_bytes,
                                       plan, write)
    return {"outputs": [o for o, _ in outs], "lines": lines, "map_lines": map_lines, "map_keys": keys,
            "device_ms": {k: t.ms() for k, t in timers.items()}}


def frappe_feature(input_dir: str, device="cuda", chunk_bytes: int = 64 << 20) -> Dict:
    """get_frape_feature.py's main: each glob(input_dir + '/*libsvm') -> path.split('.')[0] + '_.libsvm' with the
    label -1 rewritten to 0 (the reference ignores output_dir, and so does this).  Returns the outputs, line counts
    and device milliseconds."""
    dev = _device(device)
    _check_sizes(int(chunk_bytes))
    outs = frappe_outputs(input_dir)
    timer = Timer()

    def plan(text, n, info_ptr, ws_ptr, ws_bytes):
        check(_L.ctr_frappe_plan(text, n, info_ptr, ws_ptr, ws_bytes, _stream()), "ctr_frappe_plan")

    def write(text, n, out, ws_ptr, ws_bytes):
        check(_L.ctr_frappe_write(text, n, out, ws_ptr, ws_bytes, _stream()), "ctr_frappe_write")

    lines = {}
    with torch.cuda.device(dev):
        for out, ins in outs:
            with open(out, "wb") as fh:
                lines[out] = _stream_lines(ins, fh, dev, int(chunk_bytes), timer, _L.ctr_frappe_workspace_bytes, plan,
                                           write)
    return {"outputs": [o for o, _ in outs], "lines": lines, "device_ms": {"frappe": timer.ms()}}
