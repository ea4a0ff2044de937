"""REST surface of the hot-path services on werkzeug (Flask is not installed here), reproducing the
routes, JSON keys, status codes, messages and GET-URI bodies of the reference:

  POST  /projections   projection_image/server.py:72-154      201 / 409 / 406
  PATCH /fieldTypes    data_type_handler_image/server.py:40-90 200 / 406
  POST  /histograms    histogram_image/server.py:43-120        201 / 409 / 406
  GET   /files/<name>  database_api_image/server.py:52-80      paged reader (sorted by _id, limit <= 100)
  POST  /files         database_api_image/server.py:19-49      CSV ingest (the producer of the table format): body
                       {"datasetName", "datasetURI"}; 201 / 409 "duplicated dataset name" / 406 "invalid url"
                       (utils.py:78-95).  Only file:// URIs and local paths are read (no network here); rows land as
                       columns (column_store)
  POST  /models        builder_image/server.py:67-161          201 / 406: fits, evaluates and writes the predictions of
                       every classifier of "classifiersList" (builder.Builder); one URI per entry, duplicates included

Optional extension keys (absent from the reference, ignored by it): ``castTo``, ``bins``, ``range``.
The gateway paths of ``krakend/krakend.json:143-365`` map 1:1 onto these routes (INTEGRATION.md).
"""
from __future__ import annotations

import json

from werkzeug.exceptions import HTTPException
from werkzeug.routing import Map, Rule
from werkzeug.wrappers import Request, Response

from .builder import Builder
from .data_type_update import DataType
from .histogram import Histogram
from .projection import Projection
from .utils import (BuilderMetadata, BuilderRequest, Database, DataTypeMetadata, DataTypeRequest, HistogramMetadata,
                    HistogramRequest, ProjectionMetadata, ProjectionRequest)

HTTP_STATUS_CODE_SUCCESS = 200
HTTP_STATUS_CODE_SUCCESS_CREATED = 201
HTTP_STATUS_CODE_NOT_ACCEPTABLE = 406
HTTP_STATUS_CODE_CONFLICT = 409
MESSAGE_RESULT = "result"
FIRST_ARGUMENT = 0

PROJECTION_URI_GET = "/api/learningOrchestra/v1/transform/projection/"
PROJECTION_URI_PARAMS = "?query={}&limit=20&skip=0"
DATATYPE_URI_GET = "/api/learningOrchestra/v1/dataset/"
DATATYPE_URI_PARAMS = "?query={}&limit=20&skip=0"
HISTOGRAM_URI_GET = "/api/learningOrchestra/v1/explore/histogram/"
HISTOGRAM_URI_PARAMS = "?query={}&limit=10&skip=0"
BUILDER_URI_GET = "/api/learningOrchestra/v1/builder/sparkml/"
BUILDER_URI_PARAMS = "?query={}&limit=10&skip=0"

DATABASE_URL, DATABASE_REPLICA_SET, DATABASE_NAME = "mongodb://in-process", "replica_set", "database"


def _json(payload, status):
    return Response(json.dumps(payload), status=status, mimetype="application/json")


def _first_error(checks):
    """Run (validator, args, status) triples in the reference's order; first failure wins."""
    for fn, args, status in checks:
        try:
            fn(*args)
        except Exception as exc:     # the reference raises bare Exception(message)
            return _json({MESSAGE_RESULT: exc.args[FIRST_ARGUMENT]}, status)
    return None


class App:
    def __init__(self, database: Database, engine, synchronous: bool = False):
        self.database, self.engine, self.synchronous = database, engine, synchronous
        self.last_job = None            # the job the latest request started (its timings, its future)
        self.url_map = Map([
            Rule("/projections", endpoint="projection", methods=["POST"]),
            Rule("/fieldTypes", endpoint="datatype", methods=["PATCH"]),
            Rule("/histograms", endpoint="histogram", methods=["POST"]),
            Rule("/files/<filename>", endpoint="read", methods=["GET"]),
            Rule("/files", endpoint="ingest", methods=["POST"]),
            Rule("/models", endpoint="models", methods=["POST"]),
        ])

    # ---- POST /projections -----------------------------------------------------------------------------
    def on_projection(self, request):
        body = request.get_json()
        parent, out, names = body["inputDatasetName"], body["outputDatasetName"], body["names"]
        v = ProjectionRequest(self.database)
        err = _first_error([
            (v.projection_filename_validator, (out,), HTTP_STATUS_CODE_CONFLICT),
            (v.filename_validator, (parent,), HTTP_STATUS_CODE_NOT_ACCEPTABLE),
            (v.projection_fields_validator, (parent, names), HTTP_STATUS_CODE_NOT_ACCEPTABLE),
            (v.finished_processing_validator, (parent,), HTTP_STATUS_CODE_NOT_ACCEPTABLE)])
        if err is not None:
            return err
        url_in = Database.collection_database_url(DATABASE_URL, DATABASE_NAME, parent, DATABASE_REPLICA_SET)
        url_out = Database.collection_database_url(DATABASE_URL, DATABASE_NAME, out, DATABASE_REPLICA_SET)
        job = Projection(ProjectionMetadata(self.database), self.engine)
        job.create(parent, out, list(names), url_in, url_out, cast_to=body.get("castTo"), bins=body.get("bins"),
                   value_range=body.get("range"))
        self._maybe_wait(job)
        return _json({MESSAGE_RESULT: f"{PROJECTION_URI_GET}{out}{PROJECTION_URI_PARAMS}"}, HTTP_STATUS_CODE_SUCCESS_CREATED)

    # ---- PATCH /fieldTypes ------------------------------------------------------------------------------
    def on_datatype(self, request):
        body = request.get_json()
        parent, types = body["inputDatasetName"], body["types"]
        v = DataTypeRequest(self.database)
        err = _first_error([
            (v.filename_validator, (parent,), HTTP_STATUS_CODE_NOT_ACCEPTABLE),
            (v.fields_validator, (parent, types), HTTP_STATUS_CODE_NOT_ACCEPTABLE),
            (v.finished_processing_validator, (parent,), HTTP_STATUS_CODE_NOT_ACCEPTABLE)])
        if err is not None:
            return err
        job = DataType(self.database, DataTypeMetadata(self.database), self.engine)
        job.convert_existent_file(parent, types)
        self._maybe_wait(job)
        return _json({MESSAGE_RESULT: f"{DATATYPE_URI_GET}{parent}{DATATYPE_URI_PARAMS}"}, HTTP_STATUS_CODE_SUCCESS)

    # ---- POST /histograms -------------------------------------------------------------------------------
    def on_histogram(self, request):
        body = request.get_json()
        parent, out, names = body["inputDatasetName"], body["outputDatasetName"], body["names"]
        v = HistogramRequest(self.database)
        err = _first_error([
            (v.histogram_filename_validator, (out,), HTTP_STATUS_CODE_CONFLICT),
            (v.filename_validator, (parent,), HTTP_STATUS_CODE_NOT_ACCEPTABLE),
            (v.fields_validator, (parent, names), HTTP_STATUS_CODE_NOT_ACCEPTABLE),
            (v.finished_processing_validator, (parent,), HTTP_STATUS_CODE_NOT_ACCEPTABLE)])
        if err is not None:
            return err
        job = Histogram(self.database, HistogramMetadata(self.database), self.engine)
        job.create_file(parent, out, list(names), bins=body.get("bins"), value_range=body.get("range"))
        self._maybe_wait(job)
        return _json({MESSAGE_RESULT: f"{HISTOGRAM_URI_GET}{out}{HISTOGRAM_URI_PARAMS}"}, HTTP_STATUS_CODE_SUCCESS_CREATED)

    # ---- POST /models (builder_image/server.py:67-161) ------------------------------------------------------------
    def on_models(self, request):
        body = request.get_json()
        train, test, classifiers = body["trainDatasetName"], body["testDatasetName"], body["classifiersList"]
        v = BuilderRequest(self.database)
        err = _first_error([
            (v.filename_validator, (train,), HTTP_STATUS_CODE_NOT_ACCEPTABLE),
            (v.filename_validator, (test,), HTTP_STATUS_CODE_NOT_ACCEPTABLE),
            (v.model_classifiers_validator, (classifiers,), HTTP_STATUS_CODE_NOT_ACCEPTABLE),
            (v.finished_processing_validator, (train,), HTTP_STATUS_CODE_NOT_ACCEPTABLE),
            (v.finished_processing_validator, (test,), HTTP_STATUS_CODE_NOT_ACCEPTABLE)])
        if err is not None:
            return err
        url_train = Database.collection_database_url(DATABASE_URL, DATABASE_NAME, train, DATABASE_REPLICA_SET)
        url_test = Database.collection_database_url(DATABASE_URL, DATABASE_NAME, test, DATABASE_REPLICA_SET)
        job = Builder(self.database, BuilderMetadata(self.database), self.engine)
        job.build(body["modelingCode"], list(classifiers), train, test, url_train, url_test)
        self._maybe_wait(job)
        return _json({MESSAGE_RESULT: [f"{BUILDER_URI_GET}{Database.create_prediction_filename(test, c)}{BUILDER_URI_PARAMS}"
                                       for c in classifiers]}, HTTP_STATUS_CODE_SUCCESS_CREATED)

    # ---- GET /files/<name>?skip&limit&query (database_api_image/server.py:52-80) ------------------------
    def on_read(self, request, filename):
        limit, skip = 20, 0
        try:
            limit = int(request.args.get("limit", limit))
            skip = int(request.args.get("skip", skip))
        except ValueError:
            pass
        limit = min(max(limit, 0), 100) or 20
        skip = max(skip, 0)
        query = json.loads(request.args.get("query", "{}") or "{}")
        return _json({MESSAGE_RESULT: self.database.find_in_file(filename, query, skip, limit)}, HTTP_STATUS_CODE_SUCCESS)

    # ---- POST /files (database_api_image/server.py:19-49; keys constants.py:17-18; messages utils.py:79-80) ------
    def on_ingest(self, request):
        body = request.get_json()
        filename, url = body["datasetName"], body["datasetURI"]
        if filename in self.database.get_filenames():
            return _json({MESSAGE_RESULT: "duplicated dataset name"}, HTTP_STATUS_CODE_CONFLICT)
        path = url[len("file://"):] if url.startswith("file://") else url
        import os
        if not hasattr(self.database, "ingest_csv") or not os.path.isfile(path):
            return _json({MESSAGE_RESULT: "invalid url"}, HTTP_STATUS_CODE_NOT_ACCEPTABLE)
        self.database.ingest_csv(filename, path, url=url, engine=self.engine)
        return _json({MESSAGE_RESULT: f"{DATATYPE_URI_GET}{filename}?query={{}}&limit=10&skip=0"}, HTTP_STATUS_CODE_SUCCESS_CREATED)

    def _maybe_wait(self, job):
        self.last_job = job
        if self.synchronous:
            try:
                job.wait()
            except BaseException:
                pass            # like the reference, a failed job only shows as finished: False

    # ---- WSGI --------------------------------------------------------------------------------------------
    def dispatch(self, request):
        adapter = self.url_map.bind_to_environ(request.environ)
        try:
            endpoint, values = adapter.match()
            return getattr(self, f"on_{endpoint}")(request, **values)
        except HTTPException as e:
            return e

    def __call__(self, environ, start_response):
        return self.dispatch(Request(environ))(environ, start_response)


def create_app(database: Database | None = None, engine=None, synchronous: bool = False) -> App:
    if database is None:
        from .column_store import ColumnarDatabase
        database = ColumnarDatabase()
    return App(database, engine, synchronous)


def main() -> None:
    """``python -m learningorchestra_b200.server``: the routes above, ``POST /models`` included, on one werkzeug dev server
    (the reference runs one Flask process per service with ``app.run(host, port)``, e.g.
    ``projection_image/server.py:157-161``).
    LOEXEC_HOST / LOEXEC_PORT select the bind address; LOEXEC_DEVICES (e.g. "0,1,2,3"; default: every visible GPU)
    the devices — with more than one, every binned histogram / castTo projection shards the resident table over them
    (``sharding.open_engine`` -> ``lo_group_create_local``), and so does every ``POST /models`` job's frames."""
    import os

    from werkzeug.serving import run_simple

    from .sharding import open_engine

    devs = os.environ.get("LOEXEC_DEVICES") or os.environ.get("LOEXEC_DEVICE")
    engine = open_engine([int(d) for d in devs.split(",")] if devs else None)       # fails loudly without an H100
    app = create_app(None, engine)
    run_simple(os.environ.get("LOEXEC_HOST", "127.0.0.1"), int(os.environ.get("LOEXEC_PORT", "5001")), app, threaded=True)


if __name__ == "__main__":
    main()
