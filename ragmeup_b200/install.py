"""``ragmeup_b200.install()`` — make the reference's own import lines resolve to the GPU classes.

``server/RAGHelper_local.py`` / ``RAGHelper.py`` import the hot-path classes by name
(SURVEY.md §8b):

    from langchain_huggingface.embeddings import HuggingFaceEmbeddings      RAGHelper_local.py:18, RAGHelper_cloud.py:8
    from langchain_milvus.vectorstores import Milvus                         RAGHelper.py:28
    from langchain_postgres.vectorstores import PGVector                     RAGHelper.py:29
    from langchain_community.cross_encoders import HuggingFaceCrossEncoder   RAGHelper.py:12
    from ScoredCrossEncoderReranker import ScoredCrossEncoderReranker        RAGHelper.py:33
    from PostgresBM25Retriever import PostgresBM25Retriever                  RAGHelper.py:32
    from langchain.retrievers.document_compressors import FlashrankRerank   RAGHelper.py:11
        (also langchain_community.document_compressors[.flashrank_rerank])
    from langchain_community.retrievers import BM25Retriever                 RAGHelper.py:24
    from langchain.retrievers import ContextualCompressionRetriever, EnsembleRetriever   RAGHelper.py:10
    from langchain_experimental.text_splitter import SemanticChunker        RAGHelper.py:27

Calling ``install()`` before ``import RAGHelper_local`` registers same-named modules in
``sys.modules`` so those files run unchanged with ``vector_store=milvus`` (or ``postgres``).
When LangChain is installed the classes are re-based onto its abstract bases so they pass the
pydantic type checks of ``ContextualCompressionRetriever`` / ``EnsembleRetriever``; without
LangChain (this build image) the plain classes are registered.
"""
from __future__ import annotations

import importlib
import sys
import types
from typing import Any, Dict, Optional


def _module(name: str, **attrs: Any) -> types.ModuleType:
    parts = name.split(".")
    for i in range(1, len(parts) + 1):
        n = ".".join(parts[:i])
        if n not in sys.modules:
            m = types.ModuleType(n)
            m.__path__ = []  # type: ignore[attr-defined]
            sys.modules[n] = m
            if i > 1:
                setattr(sys.modules[".".join(parts[:i - 1])], parts[i - 1], m)
    mod = sys.modules[name]
    for k, v in attrs.items():
        setattr(mod, k, v)
    return mod


def build_classes() -> Dict[str, Any]:
    """The drop-in classes, re-based on LangChain's ABCs when LangChain is importable."""
    from .cross_encoder import HuggingFaceCrossEncoder
    from .embeddings import HuggingFaceEmbeddings
    from .flashrank import FlashrankRerank
    from .pg_bm25 import PostgresBM25Retriever
    from .reranker import ScoredCrossEncoderReranker
    from .retrievers import BM25Retriever, ContextualCompressionRetriever, EnsembleRetriever
    from .vectorstore import Milvus, PGVector

    out = dict(HuggingFaceEmbeddings=HuggingFaceEmbeddings, HuggingFaceCrossEncoder=HuggingFaceCrossEncoder,
               ScoredCrossEncoderReranker=ScoredCrossEncoderReranker, FlashrankRerank=FlashrankRerank,
               Milvus=Milvus, PGVector=PGVector, BM25Retriever=BM25Retriever, EnsembleRetriever=EnsembleRetriever,
               ContextualCompressionRetriever=ContextualCompressionRetriever, PostgresBM25Retriever=PostgresBM25Retriever)
    try:  # pragma: no cover - LangChain is not present in the build image
        from langchain_core.embeddings import Embeddings
        from langchain_core.vectorstores import VectorStore
        from langchain_core.documents import BaseDocumentCompressor
        from pydantic import ConfigDict
    except Exception:
        return out

    class LCEmbeddings(HuggingFaceEmbeddings, Embeddings):  # type: ignore[misc]
        pass

    def _vs(base: type) -> type:
        # keep LangChain's own as_retriever (a pydantic VectorStoreRetriever calling our search methods)
        ns = {"as_retriever": VectorStore.as_retriever, "embeddings": property(lambda self: self.embedding_func)}
        return type(base.__name__, (base, VectorStore), ns)

    from .documents import copy_document

    class LCReranker(BaseDocumentCompressor):  # type: ignore[misc]
        """pydantic form of ScoredCrossEncoderReranker (server/ScoredCrossEncoderReranker.py:12-45)."""
        model: Any
        top_n: int = 3
        model_config = ConfigDict(arbitrary_types_allowed=True, extra="forbid")

        def compress_documents(self, documents, query, callbacks=None):
            scores = self.model.score([(query, d.page_content) for d in documents])
            ranked = sorted(zip(documents, scores), key=lambda ds: ds[1], reverse=True)
            return [copy_document(d, {**d.metadata, "relevance_score": s}) for d, s in ranked[: self.top_n]]

    from . import flashrank as fr

    class LCFlashrankRerank(BaseDocumentCompressor):  # type: ignore[misc]
        """pydantic form of flashrank.FlashrankRerank (langchain-community 0.2.10's fields) [3P-recall]."""
        client: Any = None
        top_n: int = 3
        score_threshold: float = 0.0
        model: Optional[str] = None
        prefix_metadata: str = ""
        model_config = ConfigDict(arbitrary_types_allowed=True, extra="forbid")

        def __init__(self, **data: Any):
            super().__init__(**data)            # refuses unknown fields before any model is loaded
            if self.client is None:
                self.client = fr.Ranker(model_name=self.model or fr.DEFAULT_MODEL_NAME)

        def compress_documents(self, documents, query, callbacks=None):
            return fr.compress(self.client, documents, query, self.top_n, self.score_threshold, self.prefix_metadata)

        async def acompress_documents(self, documents, query, callbacks=None):
            return self.compress_documents(documents, query, callbacks)

    from langchain_core.retrievers import BaseRetriever
    from .bm25 import BM25Index
    from .retrievers import default_preprocessing_func

    class LCBM25Retriever(BaseRetriever):  # type: ignore[misc]
        """pydantic form of retrievers.BM25Retriever (GPU BM25Index behind langchain's BaseRetriever)."""
        vectorizer: Any = None
        docs: Any = None
        k: int = 4
        preprocess_func: Any = default_preprocessing_func
        model_config = ConfigDict(arbitrary_types_allowed=True)

        @classmethod
        def from_texts(cls, texts, metadatas=None, bm25_params=None, preprocess_func=default_preprocessing_func, **kwargs):
            from langchain_core.documents import Document as LCDocument
            texts = list(texts)
            if preprocess_func is default_preprocessing_func:
                vectorizer = BM25Index.from_texts(texts, **(bm25_params or {}))
            else:
                vectorizer = BM25Index([preprocess_func(t) for t in texts], **(bm25_params or {}))
            metadatas = metadatas or ({} for _ in texts)
            docs = [LCDocument(page_content=t, metadata=m) for t, m in zip(texts, metadatas)]
            return cls(vectorizer=vectorizer, docs=docs, preprocess_func=preprocess_func, **kwargs)

        @classmethod
        def from_documents(cls, documents, *, bm25_params=None, preprocess_func=default_preprocessing_func, **kwargs):
            documents = list(documents)
            return cls.from_texts([d.page_content for d in documents], [d.metadata for d in documents],
                                  bm25_params=bm25_params, preprocess_func=preprocess_func, **kwargs)

        def _get_relevant_documents(self, query, *, run_manager=None):
            return self.vectorizer.get_top_n(self.preprocess_func(query), self.docs, n=self.k)

    LCBM25Retriever.__name__ = "BM25Retriever"
    out.update(BM25Retriever=LCBM25Retriever)

    from pydantic import PrivateAttr

    class LCPostgresBM25Retriever(BaseRetriever):  # type: ignore[misc]
        """pydantic form of pg_bm25.PostgresBM25Retriever (the reference's fields; the GPU index behind them)"""
        connection_uri: Any = None
        table_name: str = "sparse_vectors"
        k: int = 4
        conn: Any = None
        cur: Any = None
        _impl: Any = PrivateAttr(default=None)
        model_config = ConfigDict(arbitrary_types_allowed=True)

        def __init__(self, **data: Any):
            super().__init__(**data)
            self._impl = PostgresBM25Retriever(connection_uri=self.connection_uri, table_name=self.table_name, k=self.k)

        def add_documents(self, documents, ids=None):
            return self._impl.add_documents(documents, ids)

        def _get_relevant_documents(self, query, *, run_manager=None):
            from langchain_core.documents import Document as LCDocument
            self._impl.k = self.k
            return [LCDocument(page_content=d.page_content, metadata=d.metadata)
                    for d in self._impl._get_relevant_documents(query)]

        def delete(self, ids):
            self._impl.delete(ids)

        def close(self):
            self._impl.close()

    LCPostgresBM25Retriever.__name__ = "PostgresBM25Retriever"
    out.update(PostgresBM25Retriever=LCPostgresBM25Retriever)
    try:   # LangChain's own fusion / compression retrievers work unchanged over BaseRetriever objects
        from langchain.retrievers import ContextualCompressionRetriever as LCC, EnsembleRetriever as LCE
        out.update(EnsembleRetriever=LCE, ContextualCompressionRetriever=LCC)
    except Exception:
        pass
    LCReranker.__name__ = "ScoredCrossEncoderReranker"
    LCFlashrankRerank.__name__ = "FlashrankRerank"
    LCEmbeddings.__name__ = "HuggingFaceEmbeddings"
    out.update(HuggingFaceEmbeddings=LCEmbeddings, Milvus=_vs(Milvus), PGVector=_vs(PGVector),
               ScoredCrossEncoderReranker=LCReranker, FlashrankRerank=LCFlashrankRerank)
    return out


_installed: Optional[Dict[str, Any]] = None


def install() -> Dict[str, Any]:
    """Register the shim modules; returns the classes that were installed."""
    global _installed
    if _installed is not None:
        return _installed
    c = build_classes()
    _module("langchain_huggingface", HuggingFaceEmbeddings=c["HuggingFaceEmbeddings"])
    _module("langchain_huggingface.embeddings", HuggingFaceEmbeddings=c["HuggingFaceEmbeddings"])
    _module("langchain_milvus", Milvus=c["Milvus"])
    _module("langchain_milvus.vectorstores", Milvus=c["Milvus"])
    _module("langchain_postgres", PGVector=c["PGVector"])
    _module("langchain_postgres.vectorstores", PGVector=c["PGVector"])
    # langchain_community is a real package when LangChain is present: only add/replace the attribute
    try:
        import langchain_community.cross_encoders as cce  # type: ignore  # pragma: no cover
        cce.HuggingFaceCrossEncoder = c["HuggingFaceCrossEncoder"]  # pragma: no cover
    except Exception:
        _module("langchain_community.cross_encoders", HuggingFaceCrossEncoder=c["HuggingFaceCrossEncoder"])
    _module("ScoredCrossEncoderReranker", ScoredCrossEncoderReranker=c["ScoredCrossEncoderReranker"])
    # vector_store=postgres: the BM25 leg (RAGHelper.py:32,445-462) runs on the GPU instead of ParadeDB
    _module("PostgresBM25Retriever", PostgresBM25Retriever=c["PostgresBM25Retriever"])
    try:
        import langchain_community.retrievers as lcr  # type: ignore  # pragma: no cover
        lcr.BM25Retriever = c["BM25Retriever"]  # pragma: no cover
    except Exception:
        _module("langchain_community.retrievers", BM25Retriever=c["BM25Retriever"])
    try:
        import langchain.retrievers  # type: ignore  # noqa: F401  # pragma: no cover
    except Exception:
        _module("langchain.retrievers", EnsembleRetriever=c["EnsembleRetriever"],
                ContextualCompressionRetriever=c["ContextualCompressionRetriever"])
    # the default reranker (RAGHelper.py:11,480).  langchain 0.2 resolves FlashrankRerank through a module
    # __getattr__; an attribute set on the real module takes precedence over it
    for name in ("langchain.retrievers.document_compressors", "langchain_community.document_compressors",
                 "langchain_community.document_compressors.flashrank_rerank"):
        try:
            mod = importlib.import_module(name)  # pragma: no cover - LangChain is not present in the build image
            mod.FlashrankRerank = c["FlashrankRerank"]  # type: ignore[attr-defined]  # pragma: no cover
        except Exception:
            _module(name, FlashrankRerank=c["FlashrankRerank"])
    # the semantic text splitter (server/RAGHelper.py:27,329-341): device embeddings + adjacent-distance kernel
    from .chunker import SemanticChunker
    c["SemanticChunker"] = SemanticChunker
    try:
        import langchain_experimental.text_splitter as lts  # type: ignore  # pragma: no cover
        lts.SemanticChunker = SemanticChunker  # pragma: no cover
    except Exception:
        _module("langchain_experimental.text_splitter", SemanticChunker=SemanticChunker)
    _installed = c
    return c
