"""Head-less play loop: the control flow of ChessGame (ChessGame.py:55-69, 153-204) without tkinter.

`python -m cchess_zero_b200.play --ai_count 2 --ai_function mcts --play_playout 400` lets the engine play itself and
prints the board after every move; with --ai_count 1 the human types moves as `x0 y0 x1 y1` board coordinates (the
tuple ChessBoard.select would have produced, ChessBoard.py:75-114)."""
import argparse
import time

from .selfplay import cchess_main


class ChessGame(object):
    """Text-mode stand-in for the reference's ChessGame: same constructor arguments, start()/perform_AI()/change_player()."""

    def __init__(self, in_ai_count, in_ai_function, in_play_playout, in_delay=0.0, in_end_delay=0.0, batch_size=128, search_threads=16,
                 processor="gpu", num_gpus=1, res_block_nums=7, human_color="b", network=None, quiet=False, strict=False,
                 priors="reference"):
        self.ai_count, self.ai_function = in_ai_count, in_ai_function
        self.delay, self.end_delay, self.quiet = in_delay, in_end_delay, quiet
        self.current_player = "w"
        self.human_color = human_color
        self.move_times = []
        self.cchess_engine = cchess_main(playout=in_play_playout, in_batch_size=batch_size, exploration=False, in_search_threads=search_threads,
                                         processor=processor, num_gpus=num_gpus, res_block_nums=res_block_nums, human_color=human_color,
                                         network=network, log_file=False, strict=strict, priors=priors)

    def perform_AI(self):  # ChessGame.py:183-195
        t0 = time.perf_counter()
        move, win_rate = self.cchess_engine.select_move(self.ai_function)
        self.move_times.append(time.perf_counter() - t0)
        return move, win_rate

    def game_over(self):  # ChessGame.py:115 -> cchess_main.check_end
        return self.cchess_engine.check_end()

    def start(self, max_moves=10000):  # ChessGame.py:55-69 + ChessView.start's loop (ChessView.py:121-132)
        n = 0
        while n < max_moves:
            ended, who = self.game_over()
            if ended:
                return who
            if self.ai_count == 2 or self.cchess_engine.game_borad.current_player != self.human_color:
                self.perform_AI()
            else:
                coord = tuple(int(t) for t in input("move (x0 y0 x1 y1): ").split())
                try:
                    self.cchess_engine.human_move(coord, self.ai_function)
                except ValueError as e:      # strict rules: the move would leave the king attacked; ask again
                    if not self.cchess_engine.strict:
                        raise
                    print(e)
                    continue
            n += 1
            if self.delay:
                time.sleep(self.delay)
        return ""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ai_count", default=2, choices=[1, 2], type=int)
    ap.add_argument("--ai_function", default="mcts", choices=["mcts", "net"])
    ap.add_argument("--play_playout", default=400, type=int)
    ap.add_argument("--delay", default=0.0, type=float)
    ap.add_argument("--res_block_nums", default=7, type=int)
    ap.add_argument("--human_color", default="b", choices=["w", "b"])
    ap.add_argument("--priors", default="reference", choices=["reference", "softmax"],
                    help="softmax: the AI searches (and, with --ai_function net, ranks moves) by the softmax of the legal moves' logits")
    a = ap.parse_args()
    # a human at the terminal expects the full rules: no self-check, mate ends the game
    g = ChessGame(a.ai_count, a.ai_function, a.play_playout, a.delay, res_block_nums=a.res_block_nums, human_color=a.human_color, strict=True,
                  priors=a.priors)
    print("result:", g.start())


if __name__ == "__main__":
    main()
