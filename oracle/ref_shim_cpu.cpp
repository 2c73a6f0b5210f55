// extern "C" shim over the reference's OWN cpu_func/rep_penalty.cpp (compiled
// from the reference checkout in place; see oracle/Makefile).  TEST INFRASTRUCTURE ONLY.
#include "cpu_func/rep_penalty.h"
extern "C" {
void ref_rep_penalty(int vocab_size, const uint64_t* seq, float* rep_mask, float penalty_max,
                     int sustain, int decay, int seq_len)
{ rep_penalty_cpu(vocab_size, seq, rep_mask, penalty_max, sustain, decay, seq_len); }
void ref_apply_rep_penalty(int vocab_size, const uint64_t* seq, float penalty_max, int sustain,
                           int decay, int seq_len, float* logits)
{ apply_rep_penalty_cpu(vocab_size, seq, penalty_max, sustain, decay, seq_len, logits); }
}
