"""Command line: ``embed`` and ``merge`` with the reference's flag spellings (distllm/cli.py:14-245).

Only the embedding path is provided; flags keep their names, short forms and defaults so existing
invocations keep working.
"""

from __future__ import annotations

from pathlib import Path
from typing import Any

import typer
from tqdm import tqdm

app = typer.Typer(add_completion=False, pretty_exceptions_show_locals=False)


@app.command()
def embed(  # noqa: PLR0913
    encoder_name: str = typer.Option(..., '--encoder_name', '-mn', help='Encoder architecture [auto].'),
    pretrained_model_name_or_path: str = typer.Option(
        ..., '--pretrained_model_name_or_path', '-m', help='The model weights to embed with.'),
    data_path: Path = typer.Option(..., '--data_path', '-d', help='Directory of the data files to embed.'),  # noqa: B008
    data_extension: str = typer.Option(..., '--data_extension', '-de', help='Extension of the data files to glob.'),
    output_path: Path = typer.Option(..., '--output_path', '-o', help='Directory to save the embeddings to.'),  # noqa: B008
    dataset_name: str = typer.Option(
        'jsonl', '--dataset_name', '-dn', help='Dataset reader [jsonl, jsonl_chunk, fasta, sequence_per_line].'),
    batch_size: int = typer.Option(1, '--batch_size', '-b', help='Batch size for generating the embeddings.'),
    chunk_batch_size: int = typer.Option(
        1, '--chunk_batch_size', '-cb', help='Batch size for chunked text within semantic chunking.'),
    buffer_size: int = typer.Option(1, '--buffer_size', '-bs', help='Buffer size for semantic chunking.'),
    pooler_name: str = typer.Option('mean', '--pooler_name', '-pn', help='Pooler [mean, last_token].'),
    embedder_name: str = typer.Option(
        'full_sequence', '--embedder_name', '-en', help='Embedder [full_sequence, semantic_chunk].'),
    writer_name: str = typer.Option('huggingface', '--writer_name', '-wn', help='Writer [huggingface, numpy].'),
    half_precision: bool = typer.Option(False, '--half_precision', '-hp', help='Return fp16 embeddings.'),
    eval_mode: bool = typer.Option(False, '--eval_mode', '-em', help='Set the model to evaluation mode.'),
    compile_model: bool = typer.Option(False, '--compile_model', '-cm', help='Accepted for compatibility.'),
    quantization: bool = typer.Option(
        False, '--quantization', '-q',
        help='Hold the weight matrices in 4-bit NF4 on the GPU (bitsandbytes NF4 arithmetic, dequantised exactly).'),
) -> None:
    """Generate embeddings for every ``*.<data_extension>`` file under ``data_path``."""
    from distllm_b200.distributed_embedding import embedding_worker

    dataset_kwargs: dict[str, Any] = {'name': dataset_name, 'batch_size': batch_size}
    if dataset_name == 'jsonl_chunk':
        dataset_kwargs['buffer_size'] = buffer_size
    encoder_kwargs = {
        'name': encoder_name,
        'pretrained_model_name_or_path': pretrained_model_name_or_path,
        'half_precision': half_precision,
        'eval_mode': eval_mode,
        'compile_model': compile_model,
        'quantization': quantization,
    }
    pooler_kwargs = {'name': pooler_name}
    embedder_kwargs: dict[str, Any] = {'name': embedder_name}
    if embedder_name == 'semantic_chunk':
        embedder_kwargs['chunk_batch_size'] = chunk_batch_size
    writer_kwargs = {'name': writer_name}

    data_files = list(data_path.glob(f'*.{data_extension}'))
    if not data_files:
        raise ValueError(f'No files found in {data_path} with extension {data_extension}')

    for data_file in tqdm(data_files):
        embedding_worker(
            input_path=data_file,
            output_dir=output_path,
            dataset_kwargs=dataset_kwargs,
            encoder_kwargs=encoder_kwargs,
            pooler_kwargs=pooler_kwargs,
            embedder_kwargs=embedder_kwargs,
            writer_kwargs=writer_kwargs,
        )


@app.command()
def merge(
    writer_name: str = typer.Option('huggingface', '--writer_name', '-wn', help='Writer [huggingface, numpy].'),
    num_proc: int = typer.Option(None, '--num_proc', '-np', help='Processes for merging (huggingface writer only).'),
    dataset_dir: Path = typer.Option(..., '--dataset_dir', '-d', help='Directory holding the per-file result sub-directories.'),  # noqa: B008
    output_dir: Path = typer.Option(..., '--output_dir', '-o', help='Where to write the merged dataset.'),  # noqa: B008
) -> None:
    """Merge the per-file result directories written by ``embed`` into one dataset."""
    from distllm_b200.embed import get_writer

    writer_kwargs: dict[str, Any] = {'name': writer_name}
    if writer_name == 'huggingface':
        writer_kwargs['num_proc'] = num_proc
    writer = get_writer(writer_kwargs)
    dataset_dirs = [p for p in sorted(dataset_dir.glob('*')) if p.is_dir()]
    output_dir.mkdir(parents=True, exist_ok=True)
    writer.merge(dataset_dirs, output_dir)


def main() -> None:
    app()


if __name__ == '__main__':
    main()
