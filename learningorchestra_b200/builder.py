"""``Builder`` — drop-in for ``builder_image/builder.py`` (same constructor, same ``build``), the job of ``POST /models``.

Reference job (``builder.py:30-170``): Spark loads the training and test datasets, runs the user's ``modelingCode`` on
them, fits each requested classifier with its defaults, evaluates it on ``features_evaluation`` when there is one and
writes its predictions of ``features_testing`` to ``<test><classifier>``.  Here the ``spark_session`` slot receives an
:class:`~learningorchestra_b200.engine.Engine` or a local :class:`~learningorchestra_b200.sharding.ShardedEngine`, the
datasets are opened as :class:`~builder_frontend.DeviceFrame` s in HBM (the test frame's text fields coded by the training
frame's dictionaries, as Spark's indexers fitted once would code them), and ``modelingCode`` runs against this project's
API (``training_df.features(...)``, ``Features.random_split(...)``), not pyspark.

Departures from the reference, on purpose: the classifiers run one after the other, and one that fails (a 3-class label
refused by "GB", say) records its exception on its own dataset while the others still finish — the reference drops the
classifiers after a failing one, because nobody observes the future that raised.  Every device table the job made is
freed when it ends, whether it succeeded or not.
"""
from __future__ import annotations

import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from .builder_frontend import METADATA_FIELDS, Features, device_frame, frame_fields
from .classifier import DecisionTreeClassifier, GBTClassifier, LogisticRegression, NaiveBayes, RandomForestClassifier
from .column_store import NumberColumn, ProbabilityColumn
from .utils import Database, record_exception

CLASSIFIERS = {"LR": LogisticRegression, "DT": DecisionTreeClassifier, "RF": RandomForestClassifier,
               "GB": GBTClassifier, "NB": NaiveBayes}


class Builder:
    METADATA_DOCUMENT_ID = 0
    DOCUMENT_ID_NAME = "_id"

    def __init__(self, database_connector, metadata_creator, spark_session):
        self.__database = database_connector
        self.__metadata_creator = metadata_creator
        self.__thread_pool = ThreadPoolExecutor()
        self.__engine = spark_session          # the slot the reference fills with a SparkSession
        self.last_job = None                   # Future of the submitted job (the reference drops it)
        self.timings: dict = {}                # wall seconds per phase of the last job: frames, modelingCode, per classifier

    def build(self, modeling_code: str, classifiers_list: list, train_filename: str, test_filename: str,
              database_url_training: str, dataset_url_test: str) -> None:
        """Creates (or replaces) one prediction dataset per distinct classifier, then runs the job on the pool."""
        classifiers_metadata = {}
        for classifier_name in dict.fromkeys(classifiers_list):
            classifiers_metadata[classifier_name] = self.__metadata_creator.create_file(classifier_name, train_filename,
                                                                                        test_filename)
        self.last_job = self.__thread_pool.submit(self.__pipeline, modeling_code, classifiers_metadata,
                                                  database_url_training, dataset_url_test)

    def wait(self, timeout=None):
        if self.last_job is not None:
            self.last_job.result(timeout)

    def __pipeline(self, modeling_code, classifiers_metadata, database_url_training, database_url_test) -> None:
        database = self.__database
        self.timings = {}
        frames = []
        try:
            try:
                if self.__engine is None:
                    raise RuntimeError("the builder needs an Engine in the spark_session slot (there is no CPU fallback)")
                t0 = time.perf_counter()
                training_df = device_frame(database, Database.collection_from_url(database_url_training), self.__engine,
                                           text=True)
                frames.append(training_df)
                testing_df = device_frame(database, Database.collection_from_url(database_url_test), self.__engine,
                                          text=True, dictionaries=training_df.dictionaries)
                frames.append(testing_df)
                t1 = time.perf_counter()
                features = self.__modeling_code_processing(modeling_code, training_df, testing_df)
                self.timings.update(frames=t1 - t0, modelingCode=time.perf_counter() - t1)
            except BaseException as exc:
                for metadata in classifiers_metadata.values():
                    record_exception(database, metadata["datasetName"], exc)
                raise
            for name, metadata in classifiers_metadata.items():
                try:
                    self.__classifier_processing(name, metadata, *features)
                except Exception as exc:           # this classifier's dataset only; the others still run
                    record_exception(database, metadata["datasetName"], exc)
        finally:
            for frame in frames:
                for made in frame.made:
                    made.release()
                frame.release()

    @staticmethod
    def __modeling_code_processing(modeling_code, training_df, testing_df):
        """``exec(modelingCode)`` with ``training_df`` and ``testing_df`` as locals and this module's globals
        (``builder.py:98-105``); the code binds ``features_training`` and ``features_testing`` (:class:`Features`) and
        ``features_evaluation`` (:class:`Features` or None)."""
        preprocessing_variables = {"training_df": training_df, "testing_df": testing_df}
        exec(modeling_code, globals(), preprocessing_variables)
        out = []
        for name in ("features_training", "features_testing", "features_evaluation"):
            if name not in preprocessing_variables:
                raise NameError(f"modelingCode did not bind {name}")
            value = preprocessing_variables[name]
            if not isinstance(value, Features) and not (name == "features_evaluation" and value is None):
                raise TypeError(f"{name} is a {type(value).__name__}, not Features"
                                + (" or None" if name == "features_evaluation" else ""))
            out.append(value)
        return out

    def __classifier_processing(self, name, metadata, features_training, features_testing, features_evaluation):
        phases = self.timings.setdefault(name, {})
        t0 = time.perf_counter()
        model = CLASSIFIERS[name]().fit(features_training)
        update = {"fitTime": time.perf_counter() - t0}
        phases["fit"] = update["fitTime"]
        if features_evaluation is not None:
            t0 = time.perf_counter()
            result = model.evaluate(features_evaluation)
            update["F1"], update["accuracy"] = str(float(result["f1"])), str(float(result["accuracy"]))
            phases["evaluate"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        predictions = model.transform(features_testing) if len(features_testing.row_ids) else None
        phases["transform"] = time.perf_counter() - t0
        try:
            t0 = time.perf_counter()
            self.__save_classifier_result(metadata["datasetName"], features_testing, predictions)
            phases["write"] = time.perf_counter() - t0
        finally:
            if predictions is not None:
                predictions.release()
        self.__database.update_one(metadata["datasetName"], update, {self.DOCUMENT_ID_NAME: self.METADATA_DOCUMENT_ID})
        self.__metadata_creator.update_finished_flag(metadata["datasetName"], True)

    def __save_classifier_result(self, filename, features, predictions) -> None:
        """``__save_classifier_result`` (``builder.py:146-170``): one row per row of ``features``, ``_id`` 1..n, holding
        the fields of the dataset the features came from, ``probability`` (a list per row) and ``prediction`` (the class
        index as a float); ``features`` and ``rawPrediction`` are not written."""
        n = len(features.row_ids)
        prob, pred = predicted_arrays(predictions, n)
        database, source = features._frame.source
        if getattr(database, "has_columns", lambda _f: False)(source):
            cols = source_columns(database, source, features.row_ids)
            cols["probability"] = ProbabilityColumn(prob)
            cols["prediction"] = NumberColumn(pred)
            self.__database.create_table(filename, np.arange(1, n + 1, dtype=np.int64), cols)
            return
        fields, rows = frame_fields(database, source)
        by_id = {d[self.DOCUMENT_ID_NAME]: d for d in rows}
        docs = []
        for i, row_id in enumerate(features.row_ids.tolist()):
            d = by_id[row_id]
            doc = {f: d.get(f) for f in fields}
            doc.update(probability=prob[i].tolist(), prediction=float(pred[i]), _id=i + 1)
            docs.append(doc)
        self.__database.insert_many_in_file(filename, docs)


def predicted_arrays(predictions, n: int) -> tuple[np.ndarray, np.ndarray]:
    """(probability float64[n, C], prediction float64[n]) of a classifier's :class:`~classifier.Predictions`, every
    shard's rows read back with one device-to-host copy each into its place (``row_ids`` order); (n x 0, n) for None."""
    if predictions is None:
        return np.zeros((n, 0), np.float64), np.zeros(n, np.float64)
    parts = predictions._parts
    nclasses = parts[0].nclasses if parts else 0
    prob, pred = np.empty((n, nclasses), np.float64), np.empty(n, np.float64)
    at = 0
    for p in parts:
        p.prob.to_numpy(0, nrows=p.n * nclasses, out=prob[at:at + p.n].reshape(-1))
        p.pred.to_numpy(0, nrows=p.n, out=pred[at:at + p.n])
        at += p.n
    return prob, pred


def source_columns(database, filename, row_ids) -> dict:
    """Every data field of a column-store dataset, in stored order, at the rows of ``row_ids``: the dataset's own
    columns when those are all its rows in order (they are immutable), else each column's ``take``."""
    ids = np.asarray(database.row_ids(filename), np.int64)
    row_ids = np.asarray(row_ids, np.int64)
    names = [f for f in database.column_names(filename) if f not in METADATA_FIELDS]
    if np.array_equal(ids, row_ids):
        return {f: database.column(filename, f) for f in names}
    order = np.argsort(ids, kind="stable")
    pos = order[np.searchsorted(ids, row_ids, sorter=order)]
    return {f: database.column(filename, f).take(pos) for f in names}
