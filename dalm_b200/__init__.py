"""dalm_b200 — H100-native drop-in for DALM's RAG-e2e / retriever-only training step.

Public surface mirrors the reference package `dalm` for this path:
  dalm_b200.models.rag_e2e_base_model.{AutoModelForRagE2E, Mode}
  dalm_b200.models.retriever_only_base_model.AutoModelForSentenceEmbedding
  dalm_b200.training.utils.train_utils.{get_cosine_sim, get_nt_xent_loss, get_nll, marginalize_log_probs,
                                         compute_marginalized_loss_from_logits, save_model_hook, load_model_hook}
  dalm_b200.training.rag_e2e.train_rage2e.train_e2e, dalm_b200.training.retriever_only.train_retriever_only.train_retriever
  dalm_b200.cli (typer app `cli`: version, train-rag-e2e, train-retriever-only)
(`import dalm` resolves to the alias package at the repo root, which re-exports these.)
"""
import logging

__version__ = "0.0.5"          # tracks the reference's dalm/__init__.py:1 so `dalm version` prints the same string

logging.basicConfig(level=logging.INFO, format="%(asctime)s - %(levelname)s - %(name)s - %(message)s")
