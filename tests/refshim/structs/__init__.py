"""TEST INFRASTRUCTURE ONLY.

Stand-in for the third-party `py-structs` package (setup.py:47 of the reference,
not a dependency of this project) so that the *unmodified* reference hot path
(multical/optimization/calibration.py etc.) can be imported to generate the
tests/golden/ fixtures.  Never imported by multical_b200 (the product) or by the test-suite.
"""
