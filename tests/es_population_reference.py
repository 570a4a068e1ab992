"""The round rule of a population's ES step (ramp_population_es_*), restated in numpy.

Group k's twin -- a single ES learner on the group's b episodes -- runs rounds until its record holds at least episodes_per_batch_k
noisy episodes and train_batch_size_k noisy env-steps.  The population runs rounds until every group has stopped; a group records
(its pairs are perturbed, its returns, lengths and act seeds kept) exactly in the rounds its twin runs."""
import numpy as np


def es_rounds(lengths, n_pairs, episodes_per_batch, train_batch_size):
    """lengths: [rounds][K][b] every episode's env-steps in each round the population ran (enough rounds for every group);
    n_pairs, episodes_per_batch, train_batch_size: [K].  Returns (records [rounds][K] bool: group k records in round r, r_k [K],
    the population's rounds)."""
    lengths = np.asarray(lengths)
    R, K = lengths.shape[:2]
    records = np.zeros((R, K), bool)
    r_k = np.zeros(K, np.int64)
    for k in range(K):
        episodes = steps = 0
        for r in range(R):
            records[r, k] = True
            nv = 2 * int(n_pairs[k])
            episodes += nv
            steps += int(lengths[r, k, :nv].sum())
            if episodes >= episodes_per_batch[k] and steps >= train_batch_size[k]:
                r_k[k] = r + 1
                break
        else:
            raise ValueError(f'group {k} needs more than {R} rounds')
    return records, r_k, int(r_k.max())
