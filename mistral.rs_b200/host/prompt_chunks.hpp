// prompt_chunks.hpp — the scheduler's prompt chunking for text prompts (REF mistralrs-core/src/pipeline/prompt_chunks.rs,
// without the multimodal features; paged_attention/scheduler.rs for the per-sequence chunk size): how a prompt is cut
// into chunks that fit a step's token budget, and which sequences' next chunks run together in one prompt step.
#pragma once

#include <cstddef>
#include <cstdint>
#include <vector>

namespace mrs {

struct PromptChunk {
  size_t start, end;   // prompt rows [start, end)
};

// each of `batch` scheduled prompts gets an equal share of the step's token budget, at least one row
inline size_t prompt_chunk_size(size_t batch, size_t budget) {
  const size_t c = batch ? budget / batch : budget;
  return c ? c : 1;
}

// rows [prefix_len, total_len) in chunks of at most chunk_size.  With block_align > 0 a chunk that would end inside a
// block ends at that block's start instead, when that still leaves the chunk non-empty: every chunk boundary but the
// prompt's end then falls on a block boundary, so a later prefix-cache lookup finds whole blocks.
inline std::vector<PromptChunk> build_prompt_chunk_plan(size_t total_len, size_t prefix_len, size_t chunk_size,
                                                        size_t block_align) {
  std::vector<PromptChunk> chunks;
  if (chunk_size == 0) chunk_size = 1;
  size_t pos = prefix_len < total_len ? prefix_len : total_len;
  while (pos < total_len) {
    size_t end = pos + chunk_size < total_len ? pos + chunk_size : total_len;
    if (block_align > 0) {
      const size_t aligned = end / block_align * block_align;
      if (aligned > pos && aligned < end) end = aligned;
    }
    chunks.push_back({pos, end});
    pos = end;
  }
  return chunks;
}

// The sequences whose next chunk runs in the next prompt step.  plan_indices[i] is the index of sequence i's next chunk
// in plans[i] (plans[i].size() when it has none left).  The first sequence with a chunk left sets the group's kind:
// final (its plan's last chunk) or not, and its chunk length.  Every sequence with a chunk left of the same finality —
// and, with require_uniform_query_len, the same length — joins.  A step never mixes final and non-final chunks, so
// either every sequence of it produces logits or none does.  Returns false when no sequence has a chunk left.
inline bool next_prompt_chunk_group(const std::vector<size_t> &plan_indices, const std::vector<std::vector<PromptChunk>> &plans,
                                    bool require_uniform_query_len, std::vector<size_t> &members, bool &is_final) {
  members.clear();
  const size_t n = plan_indices.size() < plans.size() ? plan_indices.size() : plans.size();
  size_t first = n;
  for (size_t i = 0; i < n; i++)
    if (plan_indices[i] < plans[i].size()) { first = i; break; }
  if (first == n) return false;
  const PromptChunk &c0 = plans[first][plan_indices[first]];
  is_final = plan_indices[first] + 1 == plans[first].size();
  const size_t qlen = c0.end - c0.start;
  for (size_t i = first; i < n; i++) {
    if (plan_indices[i] >= plans[i].size()) continue;
    const PromptChunk &c = plans[i][plan_indices[i]];
    if ((plan_indices[i] + 1 == plans[i].size()) != is_final) continue;
    if (require_uniform_query_len && c.end - c.start != qlen) continue;
    members.push_back(i);
  }
  return true;
}

}  // namespace mrs
