"""The five embedding operators of LOTUS on an H100 through lotus_b200 (needs an H100; there is no CPU path).

With the real `lotus` package installed the only change to an existing script is the vector store:

    import lotus, lotus_b200
    lotus.settings.configure(rm=SentenceTransformersRM(...), vs=lotus_b200.B200VS())     # was: vs=FaissVS()
    lotus_b200.install()          # optional: also routes sem_dedup / sem_cluster_by / sem_search to the streaming kernels

Here `lotus_b200` stands in for `lotus` itself and a bag-of-words hashing encoder stands in for the sentence encoder (no model files
in this image), so the similarities are lexical, not semantic.
"""
import tempfile

import pandas as pd

import lotus_b200 as lotus

lotus.settings.configure(rm=lotus.BagOfWordsRM(dim=256), vs=lotus.B200VS())

papers = pd.DataFrame({"title": [
    "Sparse attention kernels for long sequences",
    "A survey of approximate nearest neighbour search",
    "Exact nearest neighbour search on tensor cores",
    "Sourdough hydration and crumb structure",
    "Sourdough hydration and crumb structure (preprint)",
    "Bread baking with wild yeast",
    "Cache-aware k-means clustering",
]})
topics = pd.DataFrame({"topic": ["nearest neighbour search", "bread baking", "attention kernels"]})

with tempfile.TemporaryDirectory() as tmp:
    papers = papers.sem_index("title", f"{tmp}/papers")
    topics = topics.sem_index("topic", f"{tmp}/topics")

    print(papers.sem_sim_join(topics, left_on="title", right_on="topic", K=1))         # kNN join, one topic per paper
    print(papers.sem_search("title", "wild yeast bread", K=2, return_scores=True))     # top-K rows for one query
    for q, hits in zip(["wild yeast bread", "gpu kernels"], papers.sem_search("title", ["wild yeast bread", "gpu kernels"], K=1)):
        print(q, "->", hits["title"].tolist())                                          # several queries, ONE device search
    print(papers.sem_dedup("title", threshold=0.9))                                    # near-duplicate titles collapse
    print(papers.sem_cluster_by("title", 2))                                           # faiss-parity k-means, cluster_id column
    parts = papers.sem_partition_by(lotus.utils.cluster("title", 2))                   # same clustering as a partitioner
    print(parts["_lotus_partition_id"].tolist())
