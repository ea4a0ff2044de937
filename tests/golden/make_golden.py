"""Generates the R-semantics golden fixtures by EXECUTING THE REFERENCE'S OWN FILES
(``data_type_update.py`` and ``histogram.py`` import only the stdlib) against the in-memory
``MemoryDatabase`` of oracle/rsem.py.  Needs a checkout of the upstream learningOrchestra repository;
the JSON it writes is committed and is all the tests read.

    python tests/golden/make_golden.py /path/to/learningOrchestra

What is pinned by the reference's code itself: the per-document cast (every branch of
``DataType.field_converter``), the ``finished`` flag protocol, the histogram result-document shape.
What is restated inside MemoryDatabase (mongod is absent): ``$group`` equality and ``update_one``.
"""
import importlib.util
import json
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
REF = Path(sys.argv[1] if len(sys.argv) > 1 else ".") / "microservices"
sys.path.insert(0, str(ROOT))

from oracle import rsem  # noqa: E402


def load_reference(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class MetadataStandIn:
    """Same calls as ``*/utils.py`` Metadata (those files import pymongo/pytz and cannot be imported)."""

    def __init__(self, db):
        self.db = db

    def update_finished_flag(self, filename, flag):           # data_type_handler_image/utils.py:23-31
        self.db.update_one(filename, {"finished": flag}, {"_id": 0})

    update_finish_flag = update_finished_flag                 # histogram_image/utils.py:30-37

    def create_file(self, parent_filename, histogram_filename, fields):   # histogram_image/utils.py:12-28
        self.db.insert_one_in_file(histogram_filename, {
            "parentDatasetName": parent_filename, "fields": fields, "datasetName": histogram_filename,
            "type": "explore/histogram", "_id": 0, "finished": False, "timeCreated": "2026-09-21T00:00:00-00:00"})


def main():
    if not REF.exists():
        raise SystemExit(f"{REF} not found: pass the path of a learningOrchestra checkout")
    dtu = load_reference(REF / "data_type_handler_image" / "data_type_update.py", "ref_data_type_update")
    hst = load_reference(REF / "histogram_image" / "histogram.py", "ref_histogram")

    headers, docs = rsem.csv_rows_to_documents(rsem.TITANIC_HEADERS, rsem.titanic_shaped_rows())
    (HERE / "titanic_shaped_input.json").write_text(json.dumps({"headers": headers, "rows": rsem.titanic_shaped_rows()}))

    db = rsem.MemoryDatabase()
    db.insert_one_in_file("titanic", rsem.dataset_metadata("titanic", headers))
    for d in docs:
        db.insert_one_in_file("titanic", d)
    meta = MetadataStandIn(db)

    # ---- PATCH /fieldTypes: string -> number on four fields ------------------------------------------
    number_fields = {"Survived": "number", "Pclass": "number", "Age": "number", "Fare": "number"}
    job = dtu.DataType(db, meta)
    job.convert_existent_file("titanic", dict(number_fields))
    job.thread_pool.shutdown(wait=True)
    assert db.find_one("titanic", {"_id": 0})["finished"] is True
    after_number = [[d["_id"]] + [d[f] for f in number_fields] for d in db.find("titanic", {}) if d["_id"] != 0]
    (HERE / "reference_datatype_number.json").write_text(json.dumps({"fields": list(number_fields), "rows": after_number}))

    # ---- POST /histograms on the converted collection ---------------------------------------------------
    hist_fields = ["Survived", "Pclass", "Age", "Embarked", "Sex"]
    hjob = hst.Histogram(db, meta)
    hjob.create_file("titanic", "titanic_hist", list(hist_fields))
    hjob.thread_pool.shutdown(wait=True)
    (HERE / "reference_histogram.json").write_text(json.dumps({"fields": hist_fields, "documents": db.find("titanic_hist", {})}))

    # ---- number -> string on Age and Survived ----------------------------------------------------------
    job2 = dtu.DataType(db, meta)
    job2.convert_existent_file("titanic", {"Age": "string", "Survived": "string"})
    job2.thread_pool.shutdown(wait=True)
    after_string = [[d["_id"], d["Age"], d["Survived"]] for d in db.find("titanic", {}) if d["_id"] != 0]
    (HERE / "reference_datatype_string.json").write_text(json.dumps({"fields": ["Age", "Survived"], "rows": after_string}))

    # ---- per-value cast vectors (SURVEY.md §8c) through the reference's converter ---------------------
    vec_in = ["22", "0.42", "7.25", "1e3", "  5 ", "-0.0", "1_000", "nan", "inf", "-inf", "3.0", "9007199254740993",
              "1e-400", "1.7976931348623159e308", "", None, "1e22", "0.1", "-7", "+8.50",
              # what float(str) does with non-ASCII text: Unicode decimal digits and whitespace are mapped to ASCII first
              "１２", "٣.٥", "\u2003 5\u00a0", "-１e２", "१२३.५०",
              # cells far beyond the old 1024-byte device limit
              "0." + "0" * 1500 + "25", "7" + "0" * 1100 + "e-1100", " " * 1200 + "42" + " " * 900,
              "2.4703282292062327208051355972538996e-324" + "0" * 1500 + "1"]
    vdb = rsem.MemoryDatabase()
    vdb.insert_one_in_file("vec", {"_id": 0, "datasetName": "vec", "finished": True, "fields": ["v"]})
    for i, v in enumerate(vec_in, start=1):
        vdb.insert_one_in_file("vec", {"_id": i, "v": v})
    vjob = dtu.DataType(vdb, MetadataStandIn(vdb))
    vjob.convert_existent_file("vec", {"v": "number"})
    vjob.thread_pool.shutdown(wait=True)
    out_num = [d["v"] for d in vdb.find("vec", {}) if d["_id"] != 0]
    vjob = dtu.DataType(vdb, MetadataStandIn(vdb))
    vjob.convert_existent_file("vec", {"v": "string"})
    vjob.thread_pool.shutdown(wait=True)
    out_str = [d["v"] for d in vdb.find("vec", {}) if d["_id"] != 0]

    def enc(v):   # JSON has no nan/inf: tag them
        if isinstance(v, float) and v != v:
            return {"float": "nan"}
        if isinstance(v, float) and v in (float("inf"), float("-inf")):
            return {"float": "inf" if v > 0 else "-inf"}
        if isinstance(v, float):
            return {"float": repr(v)}
        if isinstance(v, int):
            return {"int": str(v)}
        return v
    (HERE / "reference_cast_vectors.json").write_text(json.dumps(
        {"in": vec_in, "number": [enc(v) for v in out_num], "back_to_string": out_str}, indent=1))

    # ---- byte table: $group value counts == 256-bin histogram (config M bridge) ----------------------
    from oracle import bsem_numpy as bn
    t = bn.synth_table_u8(20260921, 150, 0, 3000)
    cols = [0, 116, 117, 130, 149]
    bdb = rsem.MemoryDatabase()
    names = [f"px{c}" for c in cols]
    bdb.insert_one_in_file("bytes", rsem.dataset_metadata("bytes", names))
    for r in range(3000):
        d = {f"px{c}": int(t[c, r]) for c in cols}
        d["_id"] = r + 1
        bdb.insert_one_in_file("bytes", d)
    bjob = hst.Histogram(bdb, MetadataStandIn(bdb))
    bjob.create_file("bytes", "bytes_hist", list(names))
    bjob.thread_pool.shutdown(wait=True)
    (HERE / "reference_histogram_bytes.json").write_text(json.dumps(
        {"seed": 20260921, "ncols": 150, "nrows": 3000, "cols": cols, "documents": bdb.find("bytes_hist", {})}))
    print("golden fixtures written to", HERE)


if __name__ == "__main__":
    main()
