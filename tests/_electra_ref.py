"""fp32 / float64 restatement of HF ``ElectraModel`` (and of ``BertModel`` at any width) for the ELECTRA tests and
scripts/precision_table_electra.py, composed from the oracle's own helpers (oracle/encoders.py ``_ln`` / ``_linear`` /
``_mha``, looked up at call time so that the precision emulation's patches apply):

    e  = LayerNorm_E(word[ids] + pos[offset .. offset + n - 1] + type[0])
    h0 = e W_proj^T + b_proj            (only when the checkpoint has embeddings_project, i.e. E != H)

followed by BERT's post-LN layers (oracle.encoders.bert_hidden_states, whose embedding it replaces).  The readout is the
reference's: the sum of the last four hidden states, stripped to [start:end], mean for UTTERANCE."""
import numpy as np
import torch

from oracle import encoders as E


def electra_hidden_states(sd, input_ids, layers, heads, eps=1e-12, position_offset=0, dtype=torch.float32):
    """``ElectraModel(input_ids, output_hidden_states=True).hidden_states`` for one unpadded sentence (token types 0)."""
    ids = torch.as_tensor(input_ids, dtype=torch.long)
    if ids.dim() == 1:
        ids = ids[None]
    pos = torch.arange(ids.shape[1]) + position_offset
    x = (E._t(sd, "embeddings.word_embeddings.weight", dtype)[ids]
         + E._t(sd, "embeddings.token_type_embeddings.weight", dtype)[0]
         + E._t(sd, "embeddings.position_embeddings.weight", dtype)[pos])
    x = E._ln(x, sd, "embeddings.LayerNorm", eps, dtype)
    if "embeddings_project.weight" in sd:
        x = E._linear(x, sd, "embeddings_project", dtype)
    hs = [x]
    for i in range(layers):
        p = f"encoder.layer.{i}."
        q = E._linear(x, sd, p + "attention.self.query", dtype)
        k = E._linear(x, sd, p + "attention.self.key", dtype)
        v = E._linear(x, sd, p + "attention.self.value", dtype)
        a = E._linear(E._mha(q, k, v, heads), sd, p + "attention.output.dense", dtype)
        x = E._ln(x + a, sd, p + "attention.output.LayerNorm", eps, dtype)
        h = E.F.gelu(E._linear(x, sd, p + "intermediate.dense", dtype))
        h = E._linear(h, sd, p + "output.dense", dtype)
        x = E._ln(x + h, sd, p + "output.LayerNorm", eps, dtype)
        hs.append(x)
    return tuple(hs)


def electra_features(sd, input_ids, layers, heads, start=1, end=-1, feature_level="UTTERANCE", eps=1e-12,
                     dtype=torch.float32):
    """One sentence through the reference readout (extract_text_huggingface.py:222-249): the sum of the last four
    hidden states, [start:end], mean for UTTERANCE; float32 numpy."""
    hs = electra_hidden_states(sd, input_ids, layers, heads, eps=eps, dtype=dtype)
    tok = torch.stack(hs)[[-4, -3, -2, -1]].sum(0)[0, start:end].double().numpy()
    return (tok.mean(0) if feature_level == "UTTERANCE" else tok).astype(np.float32)

