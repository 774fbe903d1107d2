from .embedding import PSEmbedding, embedding_bag, embedding_bag_reference
from .embedding_collection import EmbeddingBagConfig, PSEmbeddingCollection
from .factorization_machine import PSFactorizationMachine, factorization_machine_reference
from .field_aware_factorization_machine import (PSFieldAwareFactorizationMachine,
                                                field_aware_factorization_machine_reference)
from .full_softmax import (FullSoftmaxResult, PSFullSoftmax, full_softmax, full_softmax_grad_reference,
                           full_softmax_reference, topk_dot)
from .get_gemm import gemm_nt, get_gemm, get_gemm_supported
from .hierarchical_softmax import PSHierarchicalSoftmax, hierarchical_softmax_reference
from .ps_linear import PSLinear, ps_linear
from .random_walk import Graph, random_walks, random_walks_reference
from .sampled_softmax import PSSampledSoftmax
from .topk import TOPK_MAX, topk_cosine, topk_cosine_reference

__all__ = ["get_gemm", "get_gemm_supported", "ps_linear", "PSLinear", "topk_cosine", "topk_cosine_reference",
           "TOPK_MAX", "embedding_bag", "embedding_bag_reference", "PSEmbedding",
           "EmbeddingBagConfig", "PSEmbeddingCollection", "gemm_nt", "PSSampledSoftmax",
           "full_softmax", "full_softmax_reference", "topk_dot", "FullSoftmaxResult",
           "PSFullSoftmax", "full_softmax_grad_reference", "PSHierarchicalSoftmax",
           "hierarchical_softmax_reference", "PSFactorizationMachine", "factorization_machine_reference",
           "PSFieldAwareFactorizationMachine", "field_aware_factorization_machine_reference",
           "Graph", "random_walks", "random_walks_reference"]
