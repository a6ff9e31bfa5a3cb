"""reference networks/reward_classifier.py -> serl_b200."""
from serl_b200.networks.reward_classifier import (RewardClassifier, create_classifier, load_classifier_func,  # noqa: F401
                                                  sample_classifier_batch, train_step)
