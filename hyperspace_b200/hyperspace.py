"""Hyperspace API -- same class and method names as the reference's ``python/hyperspace/hyperspace.py`` (py4j wrapper
over ``src/main/scala/com/microsoft/hyperspace/Hyperspace.scala:27-193``), backed by the GPU engine instead of Spark.

Each method runs the reference's action protocol (``actions/Action.scala:84-105``): validate -> begin (write log
id = base+1 in the transient state) -> op -> end (delete latestStable, write id = base+2 in the final state, recreate
latestStable).  ``op`` of create / refresh / optimize is ONE call into the C ABI (hs_create_index); everything else is
metadata on the file system, restated from:
  CreateAction.scala:29-100, CreateActionBase.scala:30-103, RefreshActionBase.scala:37-129, RefreshAction.scala:33-64,
  RefreshIncrementalAction.scala:45-133, RefreshQuickAction.scala:32-80, OptimizeAction.scala:57-148,
  DeleteAction / RestoreAction / VacuumAction / VacuumOutdatedAction / CancelAction.
"""
from __future__ import annotations

import os
import shutil
import uuid
from typing import Dict, List, Optional, Sequence, Tuple

from . import log_entry as LE
from .index_config import CoveringIndexConfig
from .log_entry import HyperspaceException, States
from .rules import bucket_id_of, index_signature
from .session import DataFrame, HyperspaceSession, RelationNode, list_data_files, read_parquet_schema

REFRESH_MODE_INCREMENTAL, REFRESH_MODE_FULL, REFRESH_MODE_QUICK = "incremental", "full", "quick"
OPTIMIZE_MODE_QUICK, OPTIMIZE_MODE_FULL = "quick", "full"


class NoChangesException(Exception):
    """actions/NoChangesException.scala: the action is a recorded no-op."""


def _struct_type(schema: Sequence[Tuple[str, str]]) -> dict:
    return {"type": "struct", "fields": [{"name": n, "type": t, "nullable": True, "metadata": {}} for n, t in schema]}


class _Action:
    transient_state = None
    final_state = None

    def __init__(self, log_manager: LE.IndexLogManager):
        self.log_manager = log_manager
        latest = log_manager.get_latest_id()
        self.base_id = latest if latest is not None else -1

    def validate(self) -> None:
        pass

    def log_entry(self) -> LE.IndexLogEntry:
        raise NotImplementedError

    def op(self) -> None:
        pass

    def _save(self, id_: int, entry: LE.IndexLogEntry) -> None:
        entry.timestamp = LE.now_ms()
        if not self.log_manager.write_log(id_, entry):
            raise HyperspaceException("Could not acquire proper state")

    def run(self) -> None:
        try:
            self.validate()
            e = self.log_entry()
            e.state, e.id = self.transient_state, self.base_id + 1
            self._save(self.base_id + 1, e)
            self.op()
            e = self.log_entry()
            e.state, e.id = self.final_state, self.base_id + 2
            if not self.log_manager.delete_latest_stable_log():
                raise HyperspaceException("Could not delete latest stable log")
            self._save(self.base_id + 2, e)
            self.log_manager.create_latest_stable_log(self.base_id + 2)
        except NoChangesException:
            return


class _DataAction(_Action):
    """CreateActionBase: shared by create / refresh / optimize."""

    def __init__(self, session: HyperspaceSession, log_manager, data_manager: LE.IndexDataManager):
        super().__init__(log_manager)
        self.session = session
        self.data_manager = data_manager
        latest = data_manager.get_latest_version_id()
        self.version_id = 0 if latest is None else latest + 1
        self.index_data_path = data_manager.get_path(self.version_id)
        self.tracker = LE.FileIdTracker()
        self.codec = 0

    def _resolve_codec(self) -> None:
        """The page codec of the files this action writes (spark.sql.parquet.compression.codec); raises for one the
        engine does not write, before any log entry exists."""
        self.codec = self.session.conf.parquet_compression_codec

    def _build_entry(self, name, indexed, included, num_buckets, lineage: bool, rel: RelationNode, content: LE.Content,
                     properties: Optional[Dict[str, str]] = None, update: Optional[LE.Update] = None) -> LE.IndexLogEntry:
        type_of = {n.lower(): t for n, t in rel.schema}
        # includedColumns stays the user's resolved columns; the lineage column is recorded only in `schema`, as
        # CoveringIndex.createIndexData does (index/covering/CoveringIndex.scala:152-186) -- a reference reader of this log
        # would otherwise try to resolve `_data_file_id` against the source on refresh
        inc = [c for c in included if c != LE.DATA_FILE_NAME_ID]
        schema = [(c, type_of.get(c.lower(), "long")) for c in list(indexed) + inc]
        if lineage:
            schema.append((LE.DATA_FILE_NAME_ID, "long"))
        source_content = LE.Content.from_leaf_files(rel.files, self.tracker)
        relation = LE.Relation(rel.root_paths, source_content, _struct_type(rel.schema), "parquet", {}, update)
        derived = {LE.LINEAGE_PROPERTY: str(lineage).lower(), LE.HAS_PARQUET_AS_SOURCE_FORMAT_PROPERTY: "true",
                   LE.INDEX_LOG_VERSION: str(self.base_id + 2)}
        props = {LE.HYPERSPACE_VERSION_PROPERTY: LE.HYPERSPACE_VERSION}
        props.update(properties or {})
        return LE.IndexLogEntry(name=name, indexedColumns=list(indexed), includedColumns=inc, schema=_struct_type(schema),
                                numBuckets=num_buckets, derived_properties=derived, content=content, relations=[relation],
                                signatures=[LE.Signature(LE.INDEX_SIGNATURE_PROVIDER, index_signature(rel))], properties=props)

    def _write(self, files: Sequence[Tuple[str, int, int]], indexed, included, num_buckets, lineage, out_dir, save_mode=0,
               deleted_ids: Sequence[int] = (), id_of=None) -> None:
        """The hot path: one hs_create_index call (body of CoveringIndex.write, index/covering/CoveringIndex.scala:56-71)."""
        from . import _native

        images = [_native.FileImage(path=LE.from_uri(u), file_id=(id_of(u, s, m) if id_of else -1)) for u, s, m in files]
        res, _ = self.session.gpu.create_index(images, list(indexed), [c for c in included if not (lineage and c == LE.DATA_FILE_NAME_ID)],
                                               num_buckets, out_dir=out_dir, output=_native.HS_OUT_FILES, save_mode=save_mode,
                                               lineage=lineage, deleted_file_ids=list(deleted_ids), job_uuid=str(uuid.uuid4()),
                                               compression=self.codec)
        res.free()


class CreateAction(_DataAction):
    transient_state, final_state = States.CREATING, States.ACTIVE

    def __init__(self, session, df: DataFrame, config: CoveringIndexConfig, log_manager, data_manager):
        super().__init__(session, log_manager, data_manager)
        self.df, self.config = df, config
        self.num_buckets = session.conf.num_buckets
        self.lineage = session.conf.lineage_enabled

    def validate(self) -> None:  # CreateAction.scala:50-81
        self._resolve_codec()
        if not isinstance(self.df.plan, RelationNode):
            raise HyperspaceException("Only creating index over HDFS file based scan nodes is supported. "
                                      "Source plan must be a bare relation (spark.read.parquet).")
        have = {c.lower() for c in self.df.plan.column_names}
        missing = [c for c in self.config.referencedColumns if c.lower() not in have]
        if missing:  # same first sentence as CreateAction.scala:63-65; the rest tells which columns
            raise HyperspaceException(f"Index config is not applicable to dataframe schema. Columns '{','.join(missing)}' could "
                                      f"not be resolved from available source columns '{','.join(self.df.plan.column_names)}'")
        type_of = {n.lower(): t for n, t in self.df.plan.schema}
        for c in self.config.indexedColumns:
            if type_of.get(c.lower()) == "boolean":  # filters and join keys on booleans are not handled: never readable
                raise HyperspaceException(f"Index config is not applicable: column '{c}' is boolean; boolean columns can be "
                                          "included in an index but not indexed")
        latest = self.log_manager.get_latest_log()
        if latest is not None and latest.state != States.DOESNOTEXIST:
            raise HyperspaceException(f"Another Index with name {self.config.indexName} already exists")

    def _resolved(self, cols):
        m = {c.lower(): c for c in self.df.plan.column_names}
        return [m[c.lower()] for c in cols]

    def log_entry(self):
        content = LE.Content.from_directory(self.index_data_path, LE.FileIdTracker())
        return self._build_entry(self.config.indexName, self._resolved(self.config.indexedColumns),
                                 self._resolved(self.config.includedColumns), self.num_buckets, self.lineage, self.df.plan, content)

    def op(self) -> None:  # CreateAction.scala:85
        rel = self.df.plan
        self.log_entry()  # assigns lineage ids to the source files in listing order (FileIdTracker)
        self._write(rel.files, self._resolved(self.config.indexedColumns), self._resolved(self.config.includedColumns),
                    self.num_buckets, self.lineage, self.index_data_path,
                    id_of=lambda u, s, m: self.tracker.add_file(u, s, m))


class _RefreshBase(_DataAction):
    transient_state, final_state = States.REFRESHING, States.ACTIVE

    def __init__(self, session, log_manager, data_manager):
        super().__init__(session, log_manager, data_manager)
        self.prev = log_manager.get_log(self.base_id)
        if self.prev is None:
            raise HyperspaceException("LogEntry must exist for refresh operation")
        self.tracker = self.prev.file_id_tracker()
        rel0 = self.prev.relations[0]
        files: List[Tuple[str, int, int]] = []
        for p in rel0.rootPaths:
            files.extend(list_data_files(p))
        schema = read_parquet_schema(files[0][0]) if files else [(f["name"], f["type"]) for f in rel0.dataSchema["fields"]]
        self.rel = RelationNode(list(rel0.rootPaths), files, schema)
        cur = {LE.FileInfo(u, s, m): (u, s, m) for u, s, m in files}
        orig = {f: f for f in self.prev.source_file_infos}
        self.appended = sorted(v for k, v in cur.items() if k not in orig)           # RefreshActionBase.scala:116-128
        self.deleted = sorted((f for f in orig if f not in cur), key=lambda f: f.name)  # RefreshActionBase.scala:97-108

    def validate(self) -> None:
        if self.prev.state != States.ACTIVE:
            raise HyperspaceException(f"Refresh is only supported in {States.ACTIVE} state. Current index state is {self.prev.state}")

    @property
    def lineage(self) -> bool:
        return self.prev.has_lineage_column

    def _included_without_lineage(self):
        return [c for c in self.prev.includedColumns if c != LE.DATA_FILE_NAME_ID]


class RefreshAction(_RefreshBase):
    """Full rebuild into v__=N+1 (RefreshAction.scala:33-64)."""

    def validate(self) -> None:
        super().validate()
        self._resolve_codec()
        if not self.appended and not self.deleted:
            raise NoChangesException("Refresh full aborted as no source data changed.")

    def log_entry(self):
        content = LE.Content.from_directory(self.index_data_path, LE.FileIdTracker())
        return self._build_entry(self.prev.name, self.prev.indexedColumns, self._included_without_lineage(), self.prev.numBuckets,
                                 self.lineage, self.rel, content)

    def op(self) -> None:
        self.log_entry()
        self._write(self.rel.files, self.prev.indexedColumns, self._included_without_lineage(), self.prev.numBuckets, self.lineage,
                    self.index_data_path, id_of=lambda u, s, m: self.tracker.add_file(u, s, m))


class RefreshIncrementalAction(_RefreshBase):
    """Index only the delta (RefreshIncrementalAction.scala:45-133, CoveringIndexTrait.refreshIncremental
    index/covering/CoveringIndexTrait.scala:57-106)."""

    def validate(self) -> None:
        super().validate()
        self._resolve_codec()
        if not self.appended and not self.deleted:
            raise NoChangesException("Refresh incremental aborted as no source data change found.")
        if self.deleted and not self.lineage:
            raise HyperspaceException("Index refresh (to handle deleted source data) is only supported on an index with lineage.")

    def op(self) -> None:
        self.log_entry()
        inc = self._included_without_lineage()
        mode = 0
        if self.deleted:  # rewrite the old index data without the rows of the deleted source files -> Overwrite semantics
            old_files = [LE.file_status(f) for f in self.prev.index_files]
            self._write(old_files, self.prev.indexedColumns, inc + [LE.DATA_FILE_NAME_ID], self.prev.numBuckets, False,
                        self.index_data_path, save_mode=0, deleted_ids=[f.id for f in self.deleted])
            mode = 1
        if self.appended:
            self._write(self.appended, self.prev.indexedColumns, inc, self.prev.numBuckets, self.lineage, self.index_data_path,
                        save_mode=mode, id_of=lambda u, s, m: self.tracker.add_file(u, s, m))

    def log_entry(self):
        new_content = LE.Content.from_directory(self.index_data_path, LE.FileIdTracker())
        if not self.deleted:  # UpdateMode.Merge: index = old files U new files (RefreshIncrementalAction.scala:115-128)
            merged = LE.Content(self.prev.content.root.merge(new_content.root))
        else:                 # UpdateMode.Overwrite
            merged = new_content
        return self._build_entry(self.prev.name, self.prev.indexedColumns, self._included_without_lineage(), self.prev.numBuckets,
                                 self.lineage, self.rel, merged)


class RefreshQuickAction(_RefreshBase):
    """Metadata only: record appended / deleted files; queries then use Hybrid Scan (RefreshQuickAction.scala:32-80)."""

    def validate(self) -> None:
        super().validate()
        if not self.appended and not self.deleted:
            raise NoChangesException("Refresh quick aborted as no source data change found.")
        if self.deleted and not self.lineage:
            raise HyperspaceException("Index refresh to handle deleted source data is only supported on an index with lineage.")

    def log_entry(self):
        tracker = self.tracker
        prev_rel = self.prev.relations[0]
        update = LE.Update(LE.Content.from_leaf_files(self.appended, tracker),
                           LE.Content.from_leaf_files([(f.name, f.size, f.modifiedTime) for f in self.deleted], tracker)
                           if self.deleted else None)
        e = self.prev.copy()
        rel = LE.Relation(prev_rel.rootPaths, prev_rel.content, prev_rel.dataSchema, prev_rel.fileFormat, prev_rel.options, update)
        e = e.copy(relations=[rel], signatures=[LE.Signature(LE.INDEX_SIGNATURE_PROVIDER, index_signature(self.rel))])
        return e


class OptimizeAction(_DataAction):
    """Bucket-wise compaction of small index files (OptimizeAction.scala:57-148)."""
    transient_state, final_state = States.OPTIMIZING, States.ACTIVE

    def __init__(self, session, log_manager, data_manager, mode: str):
        super().__init__(session, log_manager, data_manager)
        self.mode = mode
        self.prev = log_manager.get_log(self.base_id)
        if self.prev is None:
            raise HyperspaceException("LogEntry must exist for optimize operation")
        threshold = session.conf.optimize_file_size_threshold
        infos = self.prev.content.file_infos
        small = infos if mode.lower() == OPTIMIZE_MODE_FULL else [f for f in infos if f.size < threshold]
        by_bucket: Dict[int, List[LE.FileInfo]] = {}
        for f in small:
            by_bucket.setdefault(bucket_id_of(f.name), []).append(f)
        self.to_optimize = [f for fs in by_bucket.values() if len(fs) > 1 for f in fs]  # OptimizeAction.scala:96-114
        keep = {f.name for f in self.to_optimize}
        self.to_ignore = [f for f in infos if f.name not in keep]

    def validate(self) -> None:
        self._resolve_codec()
        if self.mode.lower() not in (OPTIMIZE_MODE_QUICK, OPTIMIZE_MODE_FULL):
            raise HyperspaceException(f"Unsupported optimize mode '{self.mode}' found.")
        if self.prev.state != States.ACTIVE:
            raise HyperspaceException(f"Optimize is only supported in {States.ACTIVE} state. Current state is {self.prev.state}.")
        if not self.to_optimize:
            raise NoChangesException("Optimize aborted as no optimizable index files smaller than "
                                     f"{self.session.conf.optimize_file_size_threshold} found.")

    def op(self) -> None:
        files = [(f.name, f.size, f.modifiedTime) for f in self.to_optimize]
        # index files of a lineage index carry `_data_file_id` (it is in the schema, not in includedColumns): re-read it as a
        # plain column so that the compacted files keep it
        inc = [c for c in self.prev.includedColumns if c != LE.DATA_FILE_NAME_ID]
        if self.prev.has_lineage_column:
            inc = inc + [LE.DATA_FILE_NAME_ID]
        self._write(files, self.prev.indexedColumns, inc, self.prev.numBuckets, False, self.index_data_path)

    def log_entry(self):
        new_content = LE.Content.from_directory(self.index_data_path, LE.FileIdTracker())
        if self.to_ignore:
            ignored = LE.Content.from_leaf_files([(f.name, f.size, f.modifiedTime) for f in self.to_ignore], LE.FileIdTracker())
            new_content = LE.Content(new_content.root.merge(ignored.root))
        return self.prev.copy(content=new_content)


class _StateFlip(_Action):
    """Delete / Restore: log-state flips only."""

    def __init__(self, log_manager, allowed_from: str, transient: str, final: str, what: str):
        super().__init__(log_manager)
        self.transient_state, self.final_state = transient, final
        self.allowed_from, self.what = allowed_from, what
        self.prev = log_manager.get_log(self.base_id)

    def validate(self) -> None:
        if self.prev is None or self.prev.state != self.allowed_from:
            cur = self.prev.state if self.prev else States.DOESNOTEXIST
            raise HyperspaceException(f"{self.what} is only supported in {self.allowed_from} state. Current state is {cur}")

    def log_entry(self):
        return self.prev.copy()


class VacuumAction(_Action):
    """Hard delete of a DELETED index (VacuumAction.scala)."""
    transient_state, final_state = States.VACUUMING, States.DOESNOTEXIST

    def __init__(self, log_manager, data_manager):
        super().__init__(log_manager)
        self.data_manager = data_manager
        self.prev = log_manager.get_log(self.base_id)

    def validate(self) -> None:
        if self.prev is None or self.prev.state != States.DELETED:
            cur = self.prev.state if self.prev else States.DOESNOTEXIST
            raise HyperspaceException(f"Vacuum is only supported in {States.DELETED} state. Current state is {cur}")

    def log_entry(self):
        return self.prev.copy()

    def op(self) -> None:
        for v in self.data_manager.get_all_version_ids():
            self.data_manager.delete(v)


class VacuumOutdatedAction(_Action):
    """On an ACTIVE index: drop data versions / files the latest entry no longer references (VacuumOutdatedAction.scala:86-120)."""
    transient_state, final_state = States.VACUUMINGOUTDATED, States.ACTIVE

    def __init__(self, log_manager, data_manager):
        super().__init__(log_manager)
        self.data_manager = data_manager
        self.prev = log_manager.get_log(self.base_id)

    def validate(self) -> None:
        if self.prev is None or self.prev.state != States.ACTIVE:
            cur = self.prev.state if self.prev else States.DOESNOTEXIST
            raise HyperspaceException(f"VacuumOutdated is only supported in {States.ACTIVE} state. Current state is {cur}.")

    def log_entry(self):
        return self.prev.copy()

    def op(self) -> None:
        used_versions = set(self.prev.index_version_dirs())
        for v in self.data_manager.get_all_version_ids():
            if v not in used_versions:
                self.data_manager.delete(v)
        # both sides canonical: the log holds abspath-normalised URIs, the data manager builds its paths from the raw
        # spark.hyperspace.system.path (relative, '//', trailing '/', '..', symlinks) -- comparing the two as strings
        # once classified every live file as outdated
        live = {os.path.realpath(LE.from_uri(f)) for f in self.prev.index_files}
        for v in used_versions:
            d = self.data_manager.get_path(v)
            if os.path.isdir(d):
                for fn in os.listdir(d):
                    p = os.path.join(d, fn)
                    if not fn.startswith(("_", ".")) and os.path.realpath(p) not in live:
                        os.remove(p)


class CancelAction(_Action):
    """Roll a stuck transient state back to the last stable state (CancelAction.scala:35-62)."""
    transient_state = States.CANCELLING

    def __init__(self, log_manager):
        super().__init__(log_manager)
        self.prev = log_manager.get_log(self.base_id)
        stable = log_manager.get_latest_stable_log()
        self.final_state = stable.state if stable else States.DOESNOTEXIST
        self.stable = stable

    def validate(self) -> None:
        if self.prev is None or self.prev.state in LE.STABLE_STATES:
            cur = self.prev.state if self.prev else States.DOESNOTEXIST
            raise HyperspaceException(f"Cancel() is not supported in stable states. Current state is {cur}")

    def log_entry(self):
        return (self.stable or self.prev).copy()


class Hyperspace:
    """python/hyperspace/hyperspace.py:9-214 / Hyperspace.scala:27-193."""

    def __init__(self, spark: HyperspaceSession):
        self.spark = spark

    # ---- helpers ------------------------------------------------------------------------------------
    def _paths(self, name: str):
        index_path = LE.PathResolver(self.spark.conf).get_index_path(name)
        return LE.IndexLogManager(index_path), LE.IndexDataManager(index_path)

    def _with_log_manager(self, name: str):
        lm, dm = self._paths(name)
        if lm.get_latest_id() is None:
            raise HyperspaceException(f"Index with name {name} could not be found")
        return lm, dm

    # ---- API ------------------------------------------------------------------------------------
    def indexes(self) -> List[Dict[str, object]]:
        """IndexStatistics summary (index/IndexStatistics.scala:58-59): one dict per index that is not DOESNOTEXIST."""
        root = LE.PathResolver(self.spark.conf).system_path
        out = []
        if os.path.isdir(root):
            for name in sorted(os.listdir(root)):
                e = LE.IndexLogManager(os.path.join(root, name)).get_latest_stable_log()
                if e is None or e.state == States.DOESNOTEXIST:
                    continue
                out.append({"name": e.name, "indexedColumns": e.indexedColumns, "includedColumns": e.includedColumns,
                            "numBuckets": e.numBuckets, "schema": e.schema, "indexLocation": os.path.join(root, name),
                            "state": e.state, "additionalStats": {"numBuckets": str(e.numBuckets)}})
        return out

    def index(self, indexName: str) -> Dict[str, object]:
        for i in self.indexes():
            if i["name"].lower() == indexName.lower():
                lm, _ = self._paths(indexName)
                e = lm.get_latest_stable_log()
                i.update({"indexContentPaths": e.index_files, "sizeInBytes": e.index_files_size_in_bytes,
                          "sourceFilesSizeInBytes": e.source_files_size_in_bytes, "logVersion": e.id,
                          "hasLineageColumn": e.has_lineage_column})
                return i
        raise HyperspaceException(f"Index with name {indexName} could not be found")

    def createIndex(self, dataFrame: DataFrame, indexConfig: CoveringIndexConfig) -> None:
        if not isinstance(indexConfig, CoveringIndexConfig):
            raise Exception("Invalid index config type: " + type(indexConfig).__name__)
        lm, dm = self._paths(indexConfig.indexName)
        CreateAction(self.spark, dataFrame, indexConfig, lm, dm).run()

    def deleteIndex(self, indexName: str) -> None:
        lm, _ = self._with_log_manager(indexName)
        _StateFlip(lm, States.ACTIVE, States.DELETING, States.DELETED, "Delete").run()

    def restoreIndex(self, indexName: str) -> None:
        lm, _ = self._with_log_manager(indexName)
        _StateFlip(lm, States.DELETED, States.RESTORING, States.ACTIVE, "Restore").run()

    def vacuumIndex(self, indexName: str) -> None:
        lm, dm = self._with_log_manager(indexName)
        latest = lm.get_latest_log()
        if latest is not None and latest.state == States.ACTIVE:  # IndexCollectionManager.scala:62-81
            VacuumOutdatedAction(lm, dm).run()
        else:
            VacuumAction(lm, dm).run()

    def refreshIndex(self, indexName: str, mode: str = REFRESH_MODE_FULL) -> None:
        lm, dm = self._with_log_manager(indexName)
        m = mode.lower()
        if m == REFRESH_MODE_INCREMENTAL:
            RefreshIncrementalAction(self.spark, lm, dm).run()
        elif m == REFRESH_MODE_FULL:
            RefreshAction(self.spark, lm, dm).run()
        elif m == REFRESH_MODE_QUICK:
            RefreshQuickAction(self.spark, lm, dm).run()
        else:
            raise HyperspaceException(f"Unsupported refresh mode '{mode}' found.")

    def optimizeIndex(self, indexName: str, mode: str = OPTIMIZE_MODE_QUICK) -> None:
        lm, dm = self._with_log_manager(indexName)
        OptimizeAction(self.spark, lm, dm, mode).run()

    def cancel(self, indexName: str) -> None:
        lm, _ = self._with_log_manager(indexName)
        CancelAction(lm).run()

    def explain(self, df: DataFrame, verbose: bool = False, redirectFunc=print) -> None:
        was = self.spark.isHyperspaceEnabled()
        self.spark.enableHyperspace()
        with_idx = df.explain()
        self.spark.disableHyperspace()
        without = df.explain()
        if was:
            self.spark.enableHyperspace()
        redirectFunc("=============================================================\nPlan with indexes:\n"
                     "=============================================================\n" + with_idx +
                     "\n\n=============================================================\nPlan without indexes:\n"
                     "=============================================================\n" + without + "\n")

    # python/hyperspace/hyperspace.py also exposes these as static helpers on the session
    @staticmethod
    def enable(spark: HyperspaceSession) -> HyperspaceSession:
        return spark.enableHyperspace()

    @staticmethod
    def disable(spark: HyperspaceSession) -> HyperspaceSession:
        return spark.disableHyperspace()

    @staticmethod
    def isEnabled(spark: HyperspaceSession) -> bool:
        return spark.isHyperspaceEnabled()
