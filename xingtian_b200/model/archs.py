"""Layer tables of the reference networks, in the engine's (name, kind, src, spec) form.

Names are the Keras/TF variable scopes of the reference so get_weights() keys match
TFVariables' (xt/model/tf_utils.py:84-102)."""

_FILTERS_PPO = {  # xt/model/model_utils.py:120-145 (out, kernel, stride)
    (84, 84): ((32, 8, 4), (32, 4, 2), (64, 3, 1)),
    (42, 42): ((32, 4, 2), (32, 4, 2), (64, 3, 1)),
    (15, 15): ((32, 5, 1), (64, 3, 1), (64, 3, 1)),
}
_FILTERS_IMPALA = {  # xt/model/atari_model.py:8-17
    (84, 84): ((16, 8, 4), (32, 4, 2), (256, 11, 1)),
    (42, 42): ((16, 4, 2), (32, 4, 2), (256, 11, 1)),
}


def _conv(cout, k, s, pad, act):
    return dict(k=k, s=s, cout=cout, pad=pad, act=act)


def _towers(state_dim, hidden_sizes, activation, share, filters):
    layers, tails = [], {}
    for prefix in (("shared",) if share else ("pi", "v")):
        src = "obs"
        for i, (cout, k, s) in enumerate(filters or ()):
            name = "{}_conv_layer_{}".format(prefix, i)       # model_utils.py:96
            layers.append((name, "conv", src, _conv(cout, k, s, "valid", activation)))
            src = name
        for i, width in enumerate(hidden_sizes):
            name = "{}_hidden_mlp_{}".format(prefix, i)      # model_utils.py:87
            layers.append((name, "dense", src, dict(n=width, act=activation)))
            src = name
        tails[prefix] = src
    return layers, tails


def _ppo_heads(layers, tails, action_dim, diag_gaussian):
    layers.append(("pi_latent", "dense", tails.get("shared", tails.get("pi")), dict(n=action_dim, act=None)))
    layers.append(("output_value", "dense", tails.get("shared", tails.get("v")), dict(n=1, act=None)))
    if diag_gaussian:
        # tf.get_variable('pi_logstd', (1, A)) is created after the Keras model (xt/model/ppo/ppo.py:75-78), so it is
        # the last variable TFVariables lists
        layers.append(("pi_logstd", "logstd", None, dict(n=action_dim)))


def ppo_cnn(state_dim, action_dim, hidden_sizes, activation, vf_share_layers, diag_gaussian=False):
    """get_cnn_backbone, xt/model/model_utils.py:49-80; diag_gaussian appends the pi_logstd variable."""
    key = tuple(state_dim[:2])
    if len(state_dim) != 3 or key not in _FILTERS_PPO:
        raise ValueError("Without default architecture for obs shape {}".format(list(state_dim)))
    layers, tails = _towers(state_dim, hidden_sizes, activation, vf_share_layers, _FILTERS_PPO[key])
    _ppo_heads(layers, tails, action_dim, diag_gaussian)
    return dict(input_dtype="uint8", state_dim=tuple(state_dim), scale=1.0 / 255.0, layers=layers,
                outputs=["pi_latent", "output_value"])


def ppo_mlp(state_dim, action_dim, hidden_sizes, activation, vf_share_layers, diag_gaussian=False):
    """get_mlp_backbone, xt/model/model_utils.py:22-46; diag_gaussian appends the pi_logstd variable."""
    layers, tails = _towers(state_dim, hidden_sizes, activation, vf_share_layers, None)
    _ppo_heads(layers, tails, action_dim, diag_gaussian)
    return dict(input_dtype="float32", state_dim=tuple(state_dim), scale=1.0, layers=layers,
                outputs=["pi_latent", "output_value"])


def impala_cnn(state_dim, action_dim):
    """ImpalaCnnOpt.create_model, xt/model/impala/impala_cnn_opt.py:115-157."""
    key = tuple(state_dim[:2])
    if len(state_dim) != 3 or key not in _FILTERS_IMPALA:
        raise ValueError("Without default architecture for obs shape {}".format(list(state_dim)))
    f = _FILTERS_IMPALA[key]
    sc = "explore_agent/"
    layers = [
        (sc + "conv2d", "conv", "obs", _conv(f[0][0], f[0][1], f[0][2], "same", "relu")),
        (sc + "conv2d_1", "conv", sc + "conv2d", _conv(f[1][0], f[1][1], f[1][2], "same", "relu")),
        (sc + "conv2d_2", "conv", sc + "conv2d_1", _conv(f[2][0], f[2][1], f[2][2], "valid", "relu")),
        (sc + "conv2d_3", "dense", sc + "conv2d_2", dict(n=action_dim, act=None)),   # 1x1 conv on a 1x1 map
        (sc + "dense", "dense", sc + "conv2d_2", dict(n=1, act=None)),
    ]
    return dict(input_dtype="uint8", state_dim=tuple(state_dim), scale=1.0 / 255.0, layers=layers,
                outputs=[sc + "conv2d_3", sc + "dense"])


def _dueling(layers, value, adv_name):
    """The dueling head (xt/model/dqn/dqn_cnn.py:55-58): adv = Dense(1) on the value stream's input, then the
    parameter-free combine Q = adv + (value - mean(value)) as the output."""
    layers.append((adv_name, "dense", layers[-1][2], dict(n=1, act=None)))
    layers.append(("dueling", "dueling", (value, adv_name), {}))
    return "dueling"


def dqn_cnn(state_dim, action_dim, dueling=False):
    """DqnCnn.create_model, xt/model/dqn/dqn_cnn.py:45-58."""
    layers = [
        ("conv2d", "conv", "obs", _conv(32, 8, 4, "valid", "relu")),
        ("conv2d_1", "conv", "conv2d", _conv(64, 4, 2, "valid", "relu")),
        ("conv2d_2", "conv", "conv2d_1", _conv(64, 3, 1, "valid", "relu")),
        ("dense", "dense", "conv2d_2", dict(n=256, act="relu")),
        ("dense_1", "dense", "dense", dict(n=action_dim, act=None)),
    ]
    out = _dueling(layers, "dense_1", "dense_2") if dueling else "dense_1"
    return dict(input_dtype="uint8", state_dim=tuple(state_dim), scale=1.0 / 255.0, layers=layers,
                outputs=[out])


def dqn_mlp(state_dim, action_dim, hidden_size, num_layers, dueling=False):
    """DqnMlp.create_model, xt/model/dqn/dqn_mlp.py:43-60."""
    layers, src = [], "obs"
    for i in range(num_layers):
        name = "dense" if i == 0 else "dense_{}".format(i)
        layers.append((name, "dense", src, dict(n=hidden_size, act="relu")))
        src = name
    value = "dense_{}".format(num_layers)
    layers.append((value, "dense", src, dict(n=action_dim, act=None)))
    out = _dueling(layers, value, "dense_{}".format(num_layers + 1)) if dueling else value
    return dict(input_dtype="float32", state_dim=tuple(state_dim), scale=1.0, layers=layers,
                outputs=[out])


def _impala_heads(layers, action_dim):
    """output_actions = Dense(A, softmax), output_value = Dense(1) on the last hidden tensor (impala_mlp.py:49-50,
    impala_cnn.py:55-56); the softmax is evaluated by the engine's kernels, so the layer itself is linear."""
    src = layers[-1][0]
    layers.append(("output_actions", "dense", src, dict(n=action_dim, act=None)))
    layers.append(("output_value", "dense", src, dict(n=1, act=None)))


def impala_keras_cnn(state_dim, action_dim):
    """ImpalaCnn.create_model, xt/model/impala/impala_cnn.py:44-59: DqnCnn's trunk, then the two heads."""
    layers = dqn_cnn(state_dim, action_dim)["layers"][:4]
    _impala_heads(layers, action_dim)
    return dict(input_dtype="uint8", state_dim=tuple(state_dim), scale=1.0 / 255.0, layers=layers,
                outputs=["output_actions", "output_value"])


def impala_mlp(state_dim, action_dim, hidden_size, num_layers):
    """ImpalaMlp.create_model, xt/model/impala/impala_mlp.py:39-55: DqnMlp's trunk, then the two heads."""
    layers = dqn_mlp(state_dim, action_dim, hidden_size, num_layers)["layers"][:num_layers]
    _impala_heads(layers, action_dim)
    return dict(input_dtype="float32", state_dim=tuple(state_dim), scale=1.0, layers=layers,
                outputs=["output_actions", "output_value"])


def muzero_cnn(state_dim, action_dim, value_support, reward_support, hidden_out=256):
    """MuzeroCnn (xt/model/muzero/muzero_cnn.py:42-67): representation, dynamics and prediction tables, in the order of
    MuzeroBase's weight list.  The softmax heads are linear here; the engine's kernels evaluate the softmax.  Within the
    prediction model Keras lists out_p before out_v: its layers are ordered by a depth-first walk from the outputs
    [out_p, out_v], not by creation (out_v is created first)."""
    if len(state_dim) != 3:
        raise ValueError("MuzeroCnn needs an image observation, got {}".format(list(state_dim)))
    a = action_dim
    rep = dict(input_dtype="uint8", state_dim=tuple(state_dim), scale=1.0 / 255.0, layers=[
        ("conv2d", "conv", "obs", _conv(32, 8, 4, "valid", "relu")),
        ("conv2d_1", "conv", "conv2d", _conv(32, 4, 2, "valid", "relu")),
        ("conv2d_2", "conv", "conv2d_1", _conv(64, 3, 1, "valid", "relu")),
        ("dense", "dense", "conv2d_2", dict(n=hidden_out, act="relu")),
    ], outputs=["dense"])
    dyn = dict(input_dtype="float32", state_dim=(hidden_out + a,), scale=1.0, layers=[
        ("dense", "dense", "obs", dict(n=256, act="relu")),
        ("dense_1", "dense", "dense", dict(n=128, act="relu")),
        ("out_h", "dense", "dense_1", dict(n=hidden_out, act="relu")),
        ("out_r", "dense", "dense_1", dict(n=reward_support, act=None)),
    ], outputs=["out_h", "out_r"])
    pred = dict(input_dtype="float32", state_dim=(hidden_out,), scale=1.0, layers=[
        ("dense", "dense", "obs", dict(n=128, act="relu")),
        ("out_p", "dense", "dense", dict(n=a, act=None)),
        ("out_v", "dense", "dense", dict(n=value_support, act=None)),
    ], outputs=["out_p", "out_v"])
    return rep, dyn, pred


def muzero_mlp(state_dim, action_dim, value_support, reward_support, hidden1=64, hidden2=4):
    """MuzeroMlp (xt/model/muzero/muzero_mlp.py:41-63): the same three models with HIDDEN1_UNITS / HIDDEN2_UNITS widths."""
    a = action_dim
    rep = dict(input_dtype="float32", state_dim=tuple(state_dim), scale=1.0, layers=[
        ("dense", "dense", "obs", dict(n=hidden1, act="relu")),
        ("dense_1", "dense", "dense", dict(n=hidden2, act="relu")),
    ], outputs=["dense_1"])
    dyn = dict(input_dtype="float32", state_dim=(hidden2 + a,), scale=1.0, layers=[
        ("dense", "dense", "obs", dict(n=hidden1, act="relu")),
        ("out_h", "dense", "dense", dict(n=hidden2, act="relu")),
        ("out_r", "dense", "dense", dict(n=reward_support, act=None)),
    ], outputs=["out_h", "out_r"])
    pred = dict(input_dtype="float32", state_dim=(hidden2,), scale=1.0, layers=[
        ("dense", "dense", "obs", dict(n=hidden1, act="relu")),
        ("out_p", "dense", "dense", dict(n=a, act=None)),
        ("out_v", "dense", "dense", dict(n=value_support, act=None)),
    ], outputs=["out_p", "out_v"])
    return rep, dyn, pred
