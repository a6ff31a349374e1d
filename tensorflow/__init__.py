"""Import shim: the reference drivers do `import tensorflow as tf` but never use
`tf.` afterwards (SURVEY.md section 8b).  There is no TensorFlow runtime on this
path; touching any attribute is an error."""


def __getattr__(name):
    raise AttributeError("tensorflow shim: the H100 path has no TensorFlow runtime (asked for tf.%s)"
                         % name)
