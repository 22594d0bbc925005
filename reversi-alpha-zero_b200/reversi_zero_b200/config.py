"""Configuration tree with the reference's field names and defaults (config.py:15-193) so that the
reference's YAML files (config/*.yml) and its own ``Config`` objects drive the H100 engine unchanged.
Only the sections the self-play path and the NBoard engine read are modelled; any object exposing the same attributes
(e.g. the reference's ``Config`` built by moke_config) is accepted everywhere in this package.

Engine-specific knobs live in ``Config.b200`` (not present in the reference): concurrent games per
GPU, seed, network implementation.
"""
import os


class _Section:
    def update(self, d):
        for k, v in (d or {}).items():
            cur = getattr(self, k, None)
            if isinstance(v, dict) and isinstance(cur, _Section):
                cur.update(v)
            else:
                setattr(self, k, v)
        return self


class Options(_Section):
    new = False


class ResourceConfig(_Section):
    """config.py:34-65"""

    def __init__(self, project_dir=None, data_dir=None):
        self.project_dir = project_dir or os.environ.get("PROJECT_DIR", os.getcwd())
        self.data_dir = data_dir or os.environ.get("DATA_DIR", os.path.join(self.project_dir, "data"))
        self.model_dir = os.environ.get("MODEL_DIR", os.path.join(self.data_dir, "model"))
        self.model_best_config_path = os.path.join(self.model_dir, "model_best_config.json")
        self.model_best_weight_path = os.path.join(self.model_dir, "model_best_weight.h5")
        self.next_generation_model_dir = os.path.join(self.model_dir, "next_generation")
        self.next_generation_model_dirname_tmpl = "model_%s"
        self.next_generation_model_config_filename = "model_config.json"
        self.next_generation_model_weight_filename = "model_weight.h5"
        self.play_data_dir = os.path.join(self.data_dir, "play_data")
        self.play_data_filename_tmpl = "play_%s.json"
        self.self_play_ggf_data_dir = os.path.join(self.data_dir, "self_play-ggf")
        self.ggf_filename_tmpl = "self_play-%s.ggf"
        self.log_dir = os.path.join(self.project_dir, "logs")
        self.main_log_path = os.path.join(self.log_dir, "main.log")
        self.tensorboard_log_dir = os.path.join(self.log_dir, "tensorboard")
        self.self_play_log_dir = os.path.join(self.tensorboard_log_dir, "self_play")
        self.force_learing_rate_file = os.path.join(self.data_dir, ".force-lr")
        self.force_simulation_num_file = os.path.join(self.data_dir, ".force-sim")
        self.self_play_game_idx_file = os.path.join(self.data_dir, ".self-play-game-idx")
        # engine-side weight hand-off (float32 blob in the layout of include/rz_engine.h)
        self.model_best_blob_path = os.path.join(self.model_dir, "model_best_weight.rzblob.npy")

    def create_directories(self):
        for d in (self.project_dir, self.data_dir, self.model_dir, self.play_data_dir, self.log_dir,
                  self.next_generation_model_dir, self.self_play_log_dir, self.self_play_ggf_data_dir):
            os.makedirs(d, exist_ok=True)


# field -> default, per section; values are the reference's (config.py:116-193)
_MODEL = dict(cnn_filter_num=256, cnn_filter_size=3, res_layer_num=10, l2_reg=1e-4, value_fc_size=256)          # :187-193
_PLAY = dict(                                                                                                     # :128-166
    simulation_num_per_move=200, share_mtcs_info_in_self_play=True, reset_mtcs_info_per_game=1, thinking_loop=10,
    required_visit_to_decide_action=400, start_rethinking_turn=8, c_puct=1, noise_eps=0.25, dirichlet_alpha=0.5,
    change_tau_turn=4, virtual_loss=3, prediction_queue_size=16, parallel_search_num=8, prediction_worker_sleep_sec=0.0001,
    wait_for_expanding_sleep_sec=0.00001, resign_threshold=-0.9, allowed_resign_turn=20, disable_resignation_rate=0.1,
    false_positive_threshold=0.05, resign_threshold_delta=0.01, policy_decay_turn=60, policy_decay_power=3,
    use_solver_turn=50, use_solver_turn_in_simulation=50, use_newest_next_generation_model=True)
_PLAY_DATA = dict(multi_process_num=16, nb_game_in_file=2, max_file_num=800, save_policy_of_tau_1=True,           # :116-125
                  enable_ggf_data=True, nb_game_in_ggf_file=100, drop_draw_game_rate=0)


def _section(name, defaults, doc):
    def init(self):
        for k, v in defaults.items():
            setattr(self, k, v)
    return type(name, (_Section,), {"__init__": init, "__doc__": doc})


ModelConfig = _section("ModelConfig", _MODEL, "network shape, config.py:187-193")
PlayDataConfig = _section("PlayDataConfig", _PLAY_DATA, "play-data files, config.py:116-125")


class PlayConfig(_Section):
    """MCTS / move-choice parameters, config.py:128-166"""

    def __init__(self):
        for k, v in _PLAY.items():
            setattr(self, k, v)
        self.schedule_of_simulation_num_per_move = [(0, 8), (300, 50), (2000, 200)]


class PlayWithHumanConfig(_Section):
    """Search settings for games against a person or another engine, config.py:74-92"""

    def __init__(self):
        self.parallel_search_num = 8
        self.noise_eps = 0
        self.change_tau_turn = 0
        self.resign_threshold = None
        self.use_newest_next_generation_model = True

    def update_play_config(self, pc):
        pc.noise_eps = self.noise_eps
        pc.change_tau_turn = self.change_tau_turn
        pc.parallel_search_num = self.parallel_search_num
        pc.resign_threshold = self.resign_threshold
        pc.use_newest_next_generation_model = self.use_newest_next_generation_model


class NBoardConfig(_Section):
    """NBoard engine, config.py:95-100"""

    def __init__(self):
        self.my_name = "RAZ"
        self.read_stdin_timeout = 0.1
        self.simulation_num_per_depth_about = 20
        self.hint_callback_per_sim = 10


class B200Config(_Section):
    """Engine knobs that have no counterpart in the reference."""

    def __init__(self):
        self.games_per_gpu = 4096   # concurrent game slots (replaces play_data.multi_process_num worker processes)
        self.seed = 20260922
        self.net_impl = 0           # RZ_NET_IMPL_AUTO
        self.weight_seed = 0        # random-init seed used when no weights exist (`--new`, agent/api.py:112-114)
        self.tensorboard = False    # write self/time, self/turn scalars like worker/self_play.py:125-129
        self.warm_start = False     # benchmark only: the first game of every slot starts mid-game (rz_engine_cfg.warm_start)
        self.warm_start_profile = None  # ... at a turn drawn with these weights (rz_engine_set_warm_start_profile)
        self.write_play_rows = False  # also write play_*.rzrows (280 B per ply) for the device-side ingest, worker/ingest.py
        self.train_from_json = False  # opt: parse play_*.json itself on the device and ignore the rows twins (worker/optimize.py)
        self.train_devices = None   # opt: CUDA ordinals of a data-parallel training group, e.g. [0, 1]; None = the one device
        self.solver_max_empties = 12  # ReversiPlayer's exact root solver: 13..this many empties go to the whole-GPU solver
        self.nboard_analyze = False  # NBoard: answer `analyze` with a retrograde analysis of the game (play_game/analysis.py)
        self.nboard_exact_hint = False  # NBoard: in solver range, `hint n` reports every move's exact value (100% lines)
        self.keep_promoted_models = False  # eval: archive every promoted blob under <model_dir>/promoted/ (worker/evaluate.py)
        self.nboard_book = None     # NBoard: an opening book (lib/book.py; path relative to the project directory) whose moves
                                    # `go` plays and `hint` reports inside the book; None = search every move
        self.nboard_book_learn = False  # NBoard: `learn` adds the game to the book (book: max_level) and writes it back


class LeagueConfig(_Section):
    """Round-robin between saved models with Elo ratings (`league` command, worker/league.py)"""

    def __init__(self):
        self.models = None          # blob paths / globs relative to the project directory, or {path:, model: {...}} mappings;
                                    # None = <model_dir>/promoted/*.rzblob.npy
        self.game_num_per_pair = 100
        self.play_config = None     # overrides of the evaluation play configuration
        self.anchor = 0             # index of the model whose rating is fixed at 0
        self.openings = None        # an opening suite (path relative to the project directory): each pair of rounds starts
                                    # from the next opening, once with each colour; None = the initial position


class OpeningsConfig(_Section):
    """Balanced opening suites for matches and leagues (`openings` command, lib/openings.py)"""

    def __init__(self):
        self.plies = 8
        self.count = 500
        self.max_abs_value = 0.2    # keep openings whose value (the network's value head, mover's view) is within this of 0
        self.seed = None            # None = b200.seed
        self.model = None           # blob path relative to the project directory (shape: the model section); None = best model
        self.path = os.path.join("data", "openings", "openings.txt")  # relative to the project directory
        self.book = None            # an opening book (lib/book.py) of `plies` plies: each opening's value is the book's
                                    # searched value instead of the value head; None = the value head


class BookConfig(_Section):
    """Opening book searched on the device (`book` command, lib/book.py)"""

    def __init__(self):
        self.plies = 8
        self.simulation_num_per_move = 400  # simulations of every leaf search
        self.seed = None            # None = b200.seed
        self.model = None           # blob path relative to the project directory (shape: the model section); None = best model
        self.path = os.path.join("data", "book", "book.npz")  # relative to the project directory
        self.extend = False         # grow or learn the book at `path` instead of building one (same model and simulations)
        self.grow_nodes = 0         # best-first expansions of leaves beyond the full width; 0 = no growth
        self.grow_batch = 256       # expansions per round (one search batch)
        self.max_level = 40         # the deepest level growth and learning may add (at most 40: 20 empties)
        self.grow_depth_cost = 0.0  # the priority's depth term: d + grow_depth_cost x (level - plies)
        self.learn = None           # GGF file globs (relative to the project directory) whose games are learned


class Config(_Section):
    def __init__(self, project_dir=None, data_dir=None):
        self.type = "default"
        self.opts = Options()
        self.resource = ResourceConfig(project_dir, data_dir)
        self.model = ModelConfig()
        self.play = PlayConfig()
        self.play_data = PlayDataConfig()
        self.play_with_human = PlayWithHumanConfig()
        self.nboard = NBoardConfig()
        self.b200 = B200Config()
        self.league = LeagueConfig()
        self.openings = OpeningsConfig()
        self.book = BookConfig()


def create_config(d=None, project_dir=None, data_dir=None):
    """Overlay a dict (e.g. yaml.safe_load of the reference's config/*.yml) on the defaults; unknown
    sections (trainer, eval, gui ...) are kept as plain attributes and ignored by the self-play path."""
    return Config(project_dir, data_dir).update(d or {})


def load_yaml(path, **kw):
    import yaml
    with open(path, "rt") as f:
        return create_config(yaml.safe_load(f), **kw)
