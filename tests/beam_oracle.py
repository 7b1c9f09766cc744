"""Beam search oracle: HF transformers 5.5.0's `_beam_search` bookkeeping (one prompt, do_sample=False, one EOS id)
restated with the same tensor operations over given per-step log-prob rows.

`log_probs(tokens, step)` returns the fp32 log-prob rows [N, V] of the running beams (`tokens`: [N, step] generated ids
of each); at step 0 every row belongs to the prompt.  Returns (sequences of generated ids [R, n] padded with
`pad`, sequences_scores [R] fp32, beam_indices [R, n] padded with -1, number of steps)."""
import torch


def beam_search(log_probs, num_beams, max_new_tokens, eos_token_id, length_penalty=1.0, early_stopping=False,
                num_return_sequences=1, pad=None):
    N, T = num_beams, max_new_tokens
    K = 2 * N
    fill = pad if pad is not None else eos_token_id
    top_num_beam_mask = torch.cat((torch.ones(N, dtype=torch.bool), torch.zeros(K - N, dtype=torch.bool)))
    running_sequences = torch.full((N, T), fill, dtype=torch.int64)
    sequences = running_sequences.clone()
    running_beam_scores = torch.zeros(N, dtype=torch.float)
    running_beam_scores[1:] = -1e9
    beam_scores = torch.full((N,), -1e9, dtype=torch.float)
    is_sent_finished = torch.zeros(N, dtype=torch.bool)
    heuristic_unsatisfied = torch.ones(1, dtype=torch.bool)
    running_beam_indices = torch.full((N, T), -1, dtype=torch.int32)
    beam_indices = running_beam_indices.clone()
    cur = 0
    steps = 0
    while True:
        lp = log_probs(running_sequences[:, :cur], cur).float()
        V = lp.shape[-1]
        steps += 1
        acc = (lp + running_beam_scores[:, None]).reshape(N * V)
        # _get_top_k_continuations
        topk_log_probs, topk_indices = torch.topk(acc, k=K)
        beam = topk_indices // V
        topk_running_beam_indices = running_beam_indices[beam].clone()
        topk_running_sequences = running_sequences[beam].clone()
        topk_ids = topk_indices % V
        topk_running_sequences[:, cur] = topk_ids
        topk_running_beam_indices[:, cur] = beam.to(torch.int32)
        # stopping criteria: EOS and max length
        hits = (topk_ids == eos_token_id) if eos_token_id is not None else torch.zeros(K, dtype=torch.bool)
        if cur + 1 >= T:
            hits = torch.ones(K, dtype=torch.bool)
        # _get_running_beams_for_next_iteration
        running_lp = topk_log_probs + hits.to(torch.float32) * -1.0e9
        nxt = torch.topk(running_lp, k=N)[1]
        running_sequences = topk_running_sequences[nxt]
        running_beam_scores = running_lp[nxt]
        running_beam_indices = topk_running_beam_indices[nxt]
        # _update_finished_beams
        did_finish = hits & top_num_beam_mask
        fin_lp = topk_log_probs / ((cur + 1) ** length_penalty)
        full = bool(is_sent_finished.all()) and early_stopping is True
        fin_lp = fin_lp + float(full) * -1.0e9
        fin_lp = fin_lp + (~heuristic_unsatisfied).to(torch.float32) * -1.0e9
        fin_lp = fin_lp + (~did_finish) * -1.0e9
        merged_scores = torch.cat((beam_scores, fin_lp))
        keep = torch.topk(merged_scores, k=N)[1]
        sequences = torch.cat((sequences, topk_running_sequences))[keep]
        beam_scores = merged_scores[keep]
        beam_indices = torch.cat((beam_indices, topk_running_beam_indices))[keep]
        is_sent_finished = torch.cat((is_sent_finished, did_finish))[keep]
        cur += 1
        # _check_early_stop_heuristic
        best_len = T if (early_stopping == "never" and length_penalty > 0.0) else cur
        best_possible = running_beam_scores[:1] / (best_len ** length_penalty)
        worst = torch.where(is_sent_finished, torch.min(beam_scores), -1.0e9)
        heuristic_unsatisfied = heuristic_unsatisfied & torch.any(best_possible > worst)
        unfinished = bool(heuristic_unsatisfied.any()) and not (bool(is_sent_finished.all()) and early_stopping is True) \
            and not bool(hits.all())
        if not unfinished:
            break
    R = num_return_sequences
    seqs, scores, idx = sequences[:R], beam_scores[:R], beam_indices[:R]
    n = int((idx + 1).bool().sum(dim=1).max())
    return seqs[:, :n], scores, idx[:, :n].to(torch.int64), steps
