"""Import-compatibility package: lets filter definitions written for commaai/rednose
(``from rednose.helpers.ekf_sym import gen_code`` ...) run unchanged on the H100-native engine.
Everything here re-exports ``rednose_b200``."""
