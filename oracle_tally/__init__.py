"""The CPU oracle's literal model selection (test infrastructure): see tally_py."""
