"""Host-side collaborators of the three hot-path services, mirroring the reference's ``utils.py``
files (same class / method names, same documents, same messages):

  * ``Database``  — the union of the reference's pymongo wrappers
    (``projection_image/utils.py:40-69``, ``histogram_image/utils.py:40-69``,
    ``data_type_handler_image/utils.py:34-57``) over an in-process document store.  MongoDB itself is
    out of scope (SURVEY.md §2); any object with these methods (e.g. a real pymongo wrapper) can be
    injected instead.  There is deliberately no ``aggregate``: the ``$group`` it served is what the GPU
    histogram replaces.
  * ``ProjectionMetadata`` / ``HistogramMetadata`` / ``DataTypeMetadata`` — the three ``Metadata``
    classes (``projection_image/utils.py:6-37``, ``histogram_image/utils.py:6-37``,
    ``data_type_handler_image/utils.py:6-31``): identical documents and call signatures.
  * ``ProjectionRequest`` / ``HistogramRequest`` / ``DataTypeRequest`` — the three ``UserRequest``
    validators with the reference's message strings (``*/utils.py`` UserRequest).
  * ``BuilderMetadata`` / ``BuilderRequest`` — the builder's ``Metadata`` and ``UserRequest``
    (``builder_image/utils.py:45-86`` and ``:89-131``), for ``POST /models``.
"""
from __future__ import annotations

import copy
import threading
from collections import OrderedDict
from datetime import datetime, timezone

METADATA_DOCUMENT_ID = 0
DOCUMENT_ID_NAME = "_id"


def _now() -> str:
    # reference: datetime.now(pytz "Etc/Greenwich").strftime("%Y-%m-%dT%H:%M:%S-00:00")
    return datetime.now(timezone.utc).strftime("%Y-%m-%dT%H:%M:%S-00:00")


def _matches(document: dict, query: dict) -> bool:
    for key, value in query.items():
        if key not in document:
            if value is None:
                continue
            return False
        if document[key] != value:
            return False
    return True


class Database:
    """In-process document store with the reference wrappers' method names."""

    def __init__(self, database_url=None, replica_set=None, database_port=None, database_name="database"):
        self.database_name = database_name
        self._collections: "OrderedDict[str, list[dict]]" = OrderedDict()
        self._versions: dict = {}
        self._lock = threading.RLock()

    def version(self, filename) -> int:
        """Bumped on every write that touches DATA rows of the collection (lets the GPU-resident column cache
        know when its copy is stale; flipping flags in the metadata document does not count)."""
        with self._lock:
            return self._versions.get(filename, 0)

    def _touch(self, filename):
        self._versions[filename] = self._versions.get(filename, 0) + 1

    # -- reads ---------------------------------------------------------------------------------------
    def get_filenames(self):
        with self._lock:
            return list(self._collections)

    def find(self, filename, query):
        with self._lock:
            return [copy.copy(d) for d in self._collections.get(filename, []) if _matches(d, query)]

    def find_one(self, filename, query):
        with self._lock:
            for d in self._collections.get(filename, []):
                if _matches(d, query):
                    return copy.deepcopy(d)
        return None

    def find_in_file(self, filename, query, skip=0, limit=10):
        """``database_api_image/utils.py:17-23``: sorted by ``_id``, then skip / limit."""
        docs = sorted(self.find(filename, query), key=lambda d: d[DOCUMENT_ID_NAME])
        return docs[skip:skip + limit]

    # -- writes --------------------------------------------------------------------------------------
    def insert_one_in_file(self, filename, json_object):
        with self._lock:
            self._collections.setdefault(filename, []).append(dict(json_object))
            if json_object.get(DOCUMENT_ID_NAME) != METADATA_DOCUMENT_ID:
                self._touch(filename)

    def insert_many_in_file(self, filename, json_objects):
        with self._lock:
            self._collections.setdefault(filename, []).extend(dict(o) for o in json_objects)
            self._touch(filename)

    def update_one(self, filename, new_value, query):
        with self._lock:
            for d in self._collections.get(filename, []):
                if _matches(d, query):
                    d.update(new_value)
                    if d.get(DOCUMENT_ID_NAME) != METADATA_DOCUMENT_ID:
                        self._touch(filename)
                    return

    def update_by_id(self, filename, updates: dict):
        """{_id: {field: value}} applied in one pass (the reference issues one ``update_one`` with a
        full-document filter per value, ``data_type_update.py:45``; the net effect is identical)."""
        with self._lock:
            for d in self._collections.get(filename, []):
                u = updates.get(d.get(DOCUMENT_ID_NAME))
                if u:
                    d.update(u)
            if updates:
                self._touch(filename)

    def delete_file(self, filename):
        with self._lock:
            self._collections.pop(filename, None)
            self._touch(filename)

    @staticmethod
    def collection_database_url(database_url, database_name, database_filename, database_replica_set):
        return f"{database_url}/{database_name}.{database_filename}" \
               f"?replicaSet={database_replica_set}&authSource=admin"

    @staticmethod
    def create_prediction_filename(parent_filename: str, classifier_name: str) -> str:
        """``builder_image/utils.py:38-41``: the dataset a classifier's predictions of ``parent_filename`` go to."""
        return f"{parent_filename}{classifier_name}"

    @staticmethod
    def collection_from_url(url: str) -> str:
        """Inverse of ``collection_database_url``: the collection name Spark would have opened."""
        tail = url.rsplit("/", 1)[-1].split("?", 1)[0]
        return tail.split(".", 1)[1] if "." in tail else tail


# ---- Metadata ------------------------------------------------------------------------------------------
class ProjectionMetadata:
    """``projection_image/utils.py:6-37``."""

    def __init__(self, database):
        self.database_connector = database
        self.metadata_document = {"_id": 0, "type": "transform/projection", "finished": False}

    def create_file(self, projection_filename, parent_filename, fields):
        metadata = self.metadata_document.copy()
        metadata["timeCreated"] = _now()
        metadata["datasetName"] = projection_filename
        metadata["parentDatasetName"] = parent_filename
        metadata["fields"] = list(fields)
        self.database_connector.insert_one_in_file(projection_filename, metadata)
        return metadata

    def update_finished_flag(self, filename, flag):
        self.database_connector.update_one(filename, {"finished": flag}, {"_id": 0})


class HistogramMetadata:
    """``histogram_image/utils.py:6-37`` (note the argument order and ``update_finish_flag``)."""

    def __init__(self, database):
        self.database_connector = database
        self.METADATA_DOCUMENT_ID = 0
        self.DOCUMENT_ID_NAME = "_id"

    def create_file(self, parent_filename, histogram_filename, fields):
        self.database_connector.insert_one_in_file(histogram_filename, {
            "parentDatasetName": parent_filename, "fields": list(fields), "datasetName": histogram_filename,
            "type": "explore/histogram", "_id": 0, "finished": False, "timeCreated": _now()})

    def update_finish_flag(self, histogram_filename, flag):
        self.database_connector.update_one(histogram_filename, {"finished": flag}, {"_id": 0})


class DataTypeMetadata:
    """``data_type_handler_image/utils.py:6-31``."""

    def __init__(self, database_connector):
        self.database_connector = database_connector

    def create_file(self, filename):
        self.database_connector.insert_one_in_file(filename, {
            "datasetName": filename, "timeCreated": _now(), "_id": 0, "finished": False,
            "type": "transform/dataType"})

    def update_finished_flag(self, filename, flag):
        self.database_connector.update_one(filename, {"finished": flag}, {"_id": 0})


class BuilderMetadata:
    """``builder_image/utils.py:45-86``: one prediction dataset per classifier, replaced when it exists."""

    def __init__(self, database):
        self.database_connector = database
        self.metadata_document = {"_id": 0, "type": "builder/sparkml", "finished": False}

    def create_file(self, classifier_name, train_filename, test_filename):
        metadata = self.metadata_document.copy()
        metadata["parentDatasetName"] = [train_filename, test_filename]
        metadata["timeCreated"] = _now()
        metadata["classifier"] = classifier_name
        metadata["datasetName"] = Database.create_prediction_filename(test_filename, classifier_name)
        self.database_connector.delete_file(metadata["datasetName"])
        self.database_connector.insert_one_in_file(metadata["datasetName"], metadata)
        return metadata

    def update_finished_flag(self, filename, flag):
        self.database_connector.update_one(filename, {"finished": flag}, {"_id": 0})


def record_exception(database, filename, exc: BaseException) -> None:
    """The reference swallows worker exceptions (unobserved Future) and leaves ``finished: False``
    forever; we keep ``finished: False`` and additionally note why (extra key, schema compatible)."""
    database.update_one(filename, {"exception": repr(exc)}, {"_id": 0})


# ---- request validators ------------------------------------------------------------------------------
class _UserRequestBase:
    MESSAGE_INVALID_FIELDS = "invalid fields"
    MESSAGE_INVALID_FILENAME = "invalid dataset name"
    MESSAGE_MISSING_FIELDS = "missing fields"
    MESSAGE_UNFINISHED_PROCESSING = "unfinished processing in input dataset"

    def __init__(self, database_connector):
        self.database = database_connector

    def filename_validator(self, filename):
        if filename not in self.database.get_filenames():
            raise Exception(self.MESSAGE_INVALID_FILENAME)

    def finished_processing_validator(self, filename):
        metadata = self.database.find_one(filename, {"datasetName": filename})
        if not metadata["finished"]:
            raise Exception(self.MESSAGE_UNFINISHED_PROCESSING)

    def _fields_exist(self, filename, fields):
        if not fields:
            raise Exception(self.MESSAGE_MISSING_FIELDS)
        metadata = self.database.find_one(filename, {"datasetName": filename})
        for field in fields:
            if field not in metadata["fields"]:
                raise Exception(self.MESSAGE_INVALID_FIELDS)


class ProjectionRequest(_UserRequestBase):
    """``projection_image/utils.py:72-114``."""
    MESSAGE_DUPLICATE_FILE = "duplicated projection name"

    def projection_filename_validator(self, projection_filename):
        if projection_filename in self.database.get_filenames():
            raise Exception(self.MESSAGE_DUPLICATE_FILE)

    def projection_fields_validator(self, filename, projection_fields):
        self._fields_exist(filename, projection_fields)


class HistogramRequest(_UserRequestBase):
    """``histogram_image/utils.py:71-113``."""
    MESSAGE_DUPLICATE_FILE = "duplicated dataset name"

    def histogram_filename_validator(self, histogram_filename):
        if histogram_filename in self.database.get_filenames():
            raise Exception(self.MESSAGE_DUPLICATE_FILE)

    def fields_validator(self, filename, fields):
        self._fields_exist(filename, fields)


class DataTypeRequest(_UserRequestBase):
    """``data_type_handler_image/utils.py:60-102``; ``"float32"`` is this build's optional extension
    (B-semantics cast on the GPU), the reference accepts only ``"number"`` and ``"string"``."""
    STRING_TYPE = "string"
    NUMBER_TYPE = "number"
    FLOAT32_TYPE = "float32"

    def fields_validator(self, filename, fields):
        self._fields_exist(filename, fields)
        for field in fields:
            if fields[field] not in (self.NUMBER_TYPE, self.STRING_TYPE, self.FLOAT32_TYPE):
                raise Exception(self.MESSAGE_INVALID_FIELDS)


class BuilderRequest(_UserRequestBase):
    """``builder_image/utils.py:89-131``, checked in ``analyse_request_errors``' order (``builder_image/server.py``)."""
    MESSAGE_INVALID_FILENAME = "invalid input dataset name"
    MESSAGE_INVALID_CLASSIFIER = "invalid classifier name"
    CLASSIFIERS = ("LR", "DT", "RF", "GB", "NB")

    def model_classifiers_validator(self, classifiers_list):
        for classifier_name in classifiers_list:
            if classifier_name not in self.CLASSIFIERS:
                raise Exception(self.MESSAGE_INVALID_CLASSIFIER)
