"""mlease_b200 -- H100-native ADMM logistic regression behind ml-ease's AdmmTrain/NaiveTrain/Test surface."""
from ._native import MleaseError, SO_PATH, lib  # noqa: F401
from .admm import (AdmmSession, Comm, World, item_model_train, item_model_train_cov, item_model_train_prior,  # noqa: F401
                   item_model_train_sparse, keyed_prior_from_fit,
                   keyed_cov_for_scoring, keyed_models_for_scoring, naive_train, naive_train_dense, naive_train_sparse, score,
                   score_keyed, score_keyed_cov, score_keyed_var, score_var, test_auc, test_loglik, test_loglik_keyed)
